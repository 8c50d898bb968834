"""The float64 checker of the forward launches: the bound arithmetic (derived in tests/test_bench_shapes.py, the bf16
mode's in tests/test_bf16_mode.py), the split-activation helpers the recorders use, and the fused warp's reference at
the kernels' fp32 tap positions."""
import torch
import torch.nn.functional as tF

from maskflownet_b200 import network, ops
from oracle import torch_ref


U = 2.0 ** -24                  # fp32 unit roundoff
EPS_Q, EPS_S = 2.0 ** -12, 2.0 ** -20
EPS_STORE = 2.0 ** -16
CONTROL_MARGIN = 3.0


def _ratio(err, scale):
    """err / scale element-wise; 0 where err is 0 (also when scale is), inf where only scale is 0."""
    return torch.where(err == 0, torch.zeros_like(err), err / scale)


def channel_slopes(C, slope, linear_prefix=0, device="cpu"):
    s = torch.full((1, C, 1, 1), float(slope), dtype=torch.float64, device=device)
    s[:, :linear_prefix] = 1.0
    return s


def activate(pre, slopes):
    return torch.where(pre > 0, pre, pre * slopes)


def judge(got, pre, slopes, bound, Q):
    """(max |got - ref| / bound, max |got - ref| / Q) with ref = activate(pre).  Where pre < -bound the result lies on
    the activation's negative side for both, so the error is scaled by the slope and the bound with it."""
    err = (got.double() - activate(pre, slopes)).abs()
    k = torch.where(pre > -bound, torch.ones_like(pre), slopes.expand_as(pre))
    return float(_ratio(err, k * bound).max()), float(_ratio(err, Q).max())


def _conv_op(transposed, stride, dilation):
    if transposed:      # the decoder's upfeat: ConvTranspose2d(kernel 4, stride 2, padding 1)
        return lambda a, k: tF.conv_transpose2d(a, k, stride=2, padding=1)
    return lambda a, k: tF.conv2d(a, k, stride=stride, padding=dilation, dilation=dilation)


def conv_terms(x, w, b, stride=1, dilation=1, transposed=False):
    """Float64 pre-activation reference, Q and S of one convolution (x, w, b float64)."""
    op = _conv_op(transposed, stride, dilation)
    bias = b.view(1, -1, 1, 1) if b is not None else 0.0
    pre = op(x, w) + bias
    Q = op(x * x, w * w).sqrt()
    S = op(x.abs(), w.abs()) + (b.abs().view(1, -1, 1, 1) if b is not None else 0.0)
    return pre, Q, S


def split_storage_term(pre, store_from):
    """Bound on the rounding of an output stored as a split activation: hi = bf16(v), lo = bf16(v - hi), both rounded to
    nearest with 8-bit significands, so |v - hi - lo| <= 2^-8 |v - hi| <= 2^-16 |v|.  Channels >= store_from (a linear
    prefix stays fp32); 0 for an fp32 output (store_from None).  In pre-activation units, so that judge's slope scaling
    applies to it as to the rest of the bound.  It matters where Q is small next to |v|: a bias-dominated output, e.g.
    a 1x1 level whose correlation input is zero but for the centre displacement."""
    if store_from is None:
        return 0.0
    t = EPS_STORE * pre.abs()
    t[:, :store_from] = 0
    return t


def conv_near_misses(x, w, b, stride=1, dilation=1, transposed=False):
    """Two wrong pre-activations the checker must reject: x and w rounded once to bf16 (no lo terms), and the first
    kernel tap dropped."""
    op = _conv_op(transposed, stride, dilation)
    bias = b.view(1, -1, 1, 1) if b is not None else 0.0
    bf = lambda t: t.to(torch.bfloat16).double()  # noqa: E731
    w_drop = w.clone()
    w_drop[:, :, 0, 0] = 0
    return {"bf16": op(bf(x), bf(w)) + bias, "tap": op(x, w_drop) + bias}


def _cout_pad(c):
    return (c + 15) // 16 * 16 if c <= 128 else 256


def _split_values(act, n, c0, c1):
    """hi + lo of channels [c0, c1) of sample n of a split activation, float64 (1, c1 - c0, H, W)."""
    one = ops.SplitAct.__new__(ops.SplitAct)
    one.channels, one.buf = act.channels, act.buf[n:n + 1]
    hi, lo = one.hi_lo()
    return hi[:, c0:c1].double() + lo[:, c0:c1].double()


def _pad_is_zero(act):
    N, C, H, W = act.shape
    G = act.buf.shape[2]
    raw = act.buf.view(torch.int16).view(N, 2, G, H, W, 8).permute(0, 1, 2, 5, 3, 4).reshape(N, 2, G * 8, H, W)
    return not bool(raw[:, :, C:].any())


def _outside_unchanged(base, before, region):
    """True when no element of `base` outside the view `region` differs bitwise from `before`."""
    inside = torch.zeros(base.shape, dtype=torch.bool, device=base.device)
    inside.as_strided(region.shape, region.stride(), region.storage_offset() - base.storage_offset()).fill_(True)
    changed = before.view(torch.int32) != base.view(torch.int32)
    return not bool((changed & ~inside).any())


def _groups_unchanged(buf, before, g0, g1):
    return torch.equal(buf[:, :, :g0], before[:, :, :g0]) and torch.equal(buf[:, :, g1:], before[:, :, g1:])


def _fp32_positions(base, d):
    """fp32 (base + d) for integer base and fp32 d, evaluated exactly in float64 and rounded once."""
    return (base + d).float().double()


def _warp_offsets(fup, scale, stride):
    """The tap offsets of the fused warp as its kernels and MXNet round them: d = fl(fl(f * scale) / stride)."""
    f = fup.double()
    return tuple(((f[:, k] * scale).float().double() / stride).float().double() for k in (0, 1))


def _warp_conv(x, fup, w, scale, stride, border, shift_y=0.0, shift_x=0.0):
    """Deformable convolution of the fused warp (no bias) at the fp32 tap positions fl((y - 1 + i) + d) computed from
    the up-sampled flow fup the kernel returned, every position then moved by (shift_y, shift_x).  float64 sums."""
    N, C, H, W = x.shape
    dy, dx = _warp_offsets(fup, scale, stride)
    ys = torch.arange(H, dtype=torch.float64, device=x.device).view(1, H, 1)
    xs = torch.arange(W, dtype=torch.float64, device=x.device).view(1, 1, W)
    out = 0
    for i in range(3):
        h = _fp32_positions(ys + (i - 1), dy) + shift_y
        for j in range(3):
            col = torch_ref.sample_tap(x, h, _fp32_positions(xs + (j - 1), dx) + shift_x, border)
            out = out + torch.einsum("fc,nchw->nfhw", w[:, :, i, j], col)
    return out


def _position_term(f, dev_y, dev_x, step=2.0 ** -16):
    """dev_y |df/dy| + dev_x |df/dx|: the error of a sampled result whose sample positions are off by up to dev_y,
    dev_x pixels.  f(sy, sx) evaluates the reference with every position moved by (sy, sx); the interpolants are
    piecewise linear, so the slopes are one-sided differences, the steeper side."""
    f0 = f(0.0, 0.0)
    sy = torch.maximum((f(step, 0.0) - f0).abs(), (f(-step, 0.0) - f0).abs()) / step
    sx = torch.maximum((f(0.0, step) - f0).abs(), (f(0.0, -step) - f0).abs()) / step
    return dev_y * sy + dev_x * sx


def _expected_convs(run):
    """3x3 convolution launches of one forward, from the graph (network.py)."""
    levels, dense = 5, len(network.DECODER_CH)
    pyramid, upfeat, context = 18, 4, 7
    # inference S: one pyramid pass over both images; per level the dense block (its last convolution carries the heads'
    # partial sums) and the heads' tail; upfeat5..2; conv5f..conv2f; dc_conv1..7
    s_inf = pyramid + levels * (dense + 1) + upfeat + 4 + context
    if run == "cascade":   # + the dual pyramid, the cascade's dense blocks + heads' tails, upfeat, context
        return s_inf + 2 * pyramid + levels * (dense + 1) + upfeat + context
    if run == "train":     # two pyramid passes; pred_flow / pred_mask (none at level 2) separately; upfeat is torch's
        return 2 * pyramid + levels * dense + (2 * 4 + 1) + 4 + context
    return s_inf


EPS_BF16_STORE = 2.0 ** -8


def _bf(t):
    return t.to(torch.bfloat16).double()


def bf16_terms(x, w, b, stride=1, dilation=1, transposed=False):
    """Float64 pre-activation and S of one convolution of the ROUNDED operands x, w (b as given)."""
    op = _conv_op(transposed, stride, dilation)
    bias = b.view(1, -1, 1, 1) if b is not None else 0.0
    pre = op(x, w) + bias
    S = op(x.abs(), w.abs()) + (b.abs().view(1, -1, 1, 1) if b is not None else 0.0)
    return pre, S


def bf16_bound(pre, S, store_from=None):
    """2^-20 S, plus the bf16 storage rounding 2^-8 |pre| on channels >= store_from (None: fp32 output)."""
    bound = EPS_S * S
    if store_from is not None:
        t = EPS_BF16_STORE * pre.abs()
        t[:, :store_from] = 0
        bound = bound + t
    return bound


def bf16_near_misses(x_full, w_full, x, w, b, stride=1, dilation=1, transposed=False):
    """The fp32-accurate result (float64 of the unrounded operands) and the rounded operands with the first tap dropped."""
    op = _conv_op(transposed, stride, dilation)
    bias = b.view(1, -1, 1, 1) if b is not None else 0.0
    w_drop = w.clone()
    w_drop[:, :, 0, 0] = 0
    return {"fp32": op(x_full, w_full) + bias, "tap": op(x, w_drop) + bias}


def _bf16_pad_is_zero(act):
    N, C, H, W = act.shape
    G = act.buf.shape[2]
    raw = act.buf.view(torch.int16).view(N, 1, G, H, W, 8).permute(0, 1, 2, 5, 3, 4).reshape(N, G * 8, H, W)
    return not bool(raw[:, C:].any())
