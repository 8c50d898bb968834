"""Every kernel launch of the benchmarked forwards against float64, at the benchmark's own shapes.

The shape of a launch decides which code runs: the split-K plan (small levels, and the short last round of a persistent
grid of one CTA per SM), the TMA box geometry of each dilation, the staged or register epilogue, the warp path.  Small
test shapes reach few of the combinations the benchmark runs, so this file runs the four benchmarked forwards once each
and checks every launch while it happens.  A recorder wraps the `ops` functions the graph calls; each wrapper runs the
original, synchronises, and compares that launch's output with a float64 reference of the same operation on the inputs
the kernel actually read (hi + lo of a split activation).  Every launch is judged on its own, so errors do not compound.
The references are plain torch in float64 on the GPU (cuDNN fp64 convolutions, oracle/torch_ref), one sample at a time.

Bound, per output element, with Q = sqrt(x^2 (*) w^2) (the scale of random rounding errors) and S = |x| (*) |w| + |b|:
    tensor-core launches (bf16 hi/lo split operands, fp32 accumulation)    |got - ref| <= 2^-12 Q + 2^-20 S
    exact-fp32 launches (SIMT warp, sampler, upsample)                      |got - ref| <= 2^-20 S
    plus, where the output is stored as a split activation (bf16 hi + lo), its rounding 2^-16 |ref| (split_storage_term).
The split's expected error is ~2^-17 Q; a bf16-only product errs by ~2^-9 Q and a dropped tap by ~Q / 3.  Where the
reference's pre-activation is below -bound the LeakyReLU scales the error by its slope, and so the bound.

Sampled operators read at positions computed in fp32.  The warp's reference computes its tap positions with the fp32
roundings of the tap-by-tap kernel and MXNet, fl((y - 1 + i) + fl(fl(f * scale) / stride)), from the up-sampled flow f
the kernel returned; the SIMT kernel rounds exactly so.  The warp through linearity samples the zero-corner operator
at the one position fl(y + d) moved by whole pixels and applies the MXNet-1.5 band correction at the per-tap positions;
where the two parts cancel (taps in the one-pixel bands) their rounding differences do not.  Its bound adds the position
deviation 2^-22 (|p| + |d| + 2) px per axis (p the pixel, d the displacement) times the slope of each part: twice the
zero-corner operator's plus the MXNet operator's.  The image warp rounds p + d after an fp32 Upsample(4); its bound adds
2^-20 (|p| + |d| + 1) px per axis times the reference's slope.  Slopes are one-sided differences, the steeper side.

The checker's sensitivity is asserted: on one real launch of each kind (fp32 NCHW, split in / split out, depth-to-space,
linear prefix, dilation >= 4) it must reject, by at least 3x, x and w rounded once to bf16 and one dropped tap.
test_checker_separates_kernel_arithmetic_from_near_misses checks the same on the CPU with the kernel's arithmetic
emulated.  Coverage is asserted too: the number of checked convolutions equals the graph's, each launch ran the kernel
variant its Cout selects, the cascade's level-2 split-K tail with split output ran, the TMA input ran at dilations
1, 2, 4, 8 and 16, and the cascade's level-6 warp ran through linearity at F = 196.

One line per launch is printed (pytest -s): op, layer, kernel, shape, dilation / stride, split-K workspace bytes, max
err / Q and max err / bound.  Not checked here: the transposed convolutions of the training graph (torch autograd).
"""
import inspect
import os
import sys
import time

import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import _lib, network, ops
from oracle import torch_ref

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
from make_golden import named_init, seeded_images  # noqa: E402

EPS_Q, EPS_S = 2.0 ** -12, 2.0 ** -20
EPS_STORE = 2.0 ** -16
CONTROL_MARGIN = 3.0


# ------------------------------------------------------------------------------------------------------------------
# the checker (any device)
# ------------------------------------------------------------------------------------------------------------------
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


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound accepts the kernel's arithmetic and rejects its near misses
# ------------------------------------------------------------------------------------------------------------------
def test_checker_separates_kernel_arithmetic_from_near_misses():
    """The widest decoder layer (dc_conv1 at level 2: 579 -> 128), small image: the kernel's arithmetic (x and w split
    into bf16 hi + lo; hi*hi + hi*lo + lo*hi, each term accumulated in fp32) passes the bound, a bf16-only result and a
    dropped tap fail it by more than CONTROL_MARGIN."""
    g = torch.Generator().manual_seed(5)
    Cin, Cout, H, W = 579, 128, 10, 18
    a = torch.randn((1, Cin, H, W), generator=g)
    x = torch.where(a > 0, a, 0.1 * a)
    w = named_init("dc_conv1.weight", (Cout, Cin, 3, 3))
    b = named_init("dc_conv1.bias", (Cout,))

    def split(t):
        hi = t.bfloat16().float()
        return hi, (t - hi).bfloat16().float()
    (xh, xl), (wh, wl) = split(x), split(w)
    conv32 = lambda p, q: tF.conv2d(p, q, padding=1)  # noqa: E731
    kern = tF.leaky_relu(conv32(xh, wh) + conv32(xh, wl) + conv32(xl, wh) + b.view(1, -1, 1, 1), 0.1)

    pre, Q, S = conv_terms(x.double(), w.double(), b.double())
    bound = EPS_Q * Q + EPS_S * S
    sl = channel_slopes(Cout, 0.1)
    ratio, err_q = judge(kern, pre, sl, bound, Q)
    assert ratio <= 1.0 and err_q < 2.0 ** -14, (ratio, err_q)
    for name, alt in conv_near_misses(x.double(), w.double(), b.double()).items():
        r, _ = judge(activate(alt, sl), pre, sl, bound, Q)
        assert r >= CONTROL_MARGIN, (name, r)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the recorder
# ------------------------------------------------------------------------------------------------------------------
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


class Recorder:
    """Wraps the ops functions of the inference and training graphs; checks every launch as it happens."""

    KINDS = ("fp32", "split", "d2s", "lin", "dil>=4")

    def __init__(self, monkeypatch, run):
        self.run, self.rows, self.failures = run, [], []
        self.packs, self.names, self.controls = {}, {}, {}
        self.orig = {}
        for name in ("conv3x3_pack", "conv_transpose4x4_pack", "conv3x3_slices", "conv3x3_split", "correlation",
                     "warp_mask", "upsample", "image_warp_concat"):
            self.orig[name] = getattr(ops, name)
            monkeypatch.setattr(ops, name, getattr(self, name))
        self.orig["pack"] = ops.SplitAct.pack
        rec = self

        def pack(act, src, c0):
            rec.split_pack(act, src, c0)
        monkeypatch.setattr(ops.SplitAct, "pack", pack)
        self.orig["_packed"], self.orig["_packed_fn"] = network._FlowNetBase._packed, network._FlowNetBase._packed_fn

        def _packed(model, name):
            p = rec.orig["_packed"](model, name)
            rec.names[p.data_ptr()] = rec._model_prefix(model) + name
            return p

        def _packed_fn(model, key, params, build):
            res = rec.orig["_packed_fn"](model, key, params, build)
            rec.names[(res[0] if isinstance(res, tuple) else res).data_ptr()] = rec._model_prefix(model) + key
            return res
        monkeypatch.setattr(network._FlowNetBase, "_packed", _packed)
        monkeypatch.setattr(network._FlowNetBase, "_packed_fn", _packed_fn)

    @staticmethod
    def _model_prefix(model):
        return "S." if isinstance(model, network.MaskFlownetS) else "cascade."

    def _bind(self, name, args, kw):
        ba = inspect.signature(self.orig[name]).bind(*args, **kw)
        ba.apply_defaults()
        return ba.arguments

    def _fail(self, msg):
        self.failures.append(f"{self.run}: {msg}")

    # ---- weight images: which fp32 weight each packed image holds ---------------------------------------------
    def conv3x3_pack(self, weight):
        packed = self.orig["conv3x3_pack"](weight)
        self.packs[packed.data_ptr()] = (weight.detach().clone(), False)
        return packed

    def conv_transpose4x4_pack(self, weight):
        packed = self.orig["conv_transpose4x4_pack"](weight)
        self.packs[packed.data_ptr()] = (weight.detach().clone(), True)
        return packed

    # ---- convolutions -----------------------------------------------------------------------------------------
    def _check_conv(self, op, packed, bias, Cout, slope, dil, stride, d2s, lp, x_of, got_of, N, Cin, H, W, ws, kern,
                    tags, store_from=None):
        w, transposed = self.packs[packed.data_ptr()]
        name = self.names.get(packed.data_ptr(), "?")
        assert transposed == d2s, name
        w = w.double()
        b = bias.detach().double() if bias is not None else None
        F = Cout // 4 if d2s else Cout
        sl = channel_slopes(F, slope, lp, w.device)
        worst, worst_q = 0.0, 0.0
        with torch.no_grad():
            for n in range(N):
                x = x_of(n)
                pre, Q, S = conv_terms(x, w, b, stride, dil, transposed)
                bound = EPS_Q * Q + EPS_S * S + split_storage_term(pre, store_from)
                r, rq = judge(got_of(n), pre, sl, bound, Q)
                worst, worst_q = max(worst, r), max(worst_q, rq)
                for tag in tags:
                    if tag not in self.controls:
                        self.controls[tag] = (name, {k: judge(activate(v, sl), pre, sl, bound, Q)[0]
                                                     for k, v in conv_near_misses(x, w, b, stride, dil, transposed).items()})
                del x, pre, Q, S, bound
        want = "conv3x3_wgmma_reduce_kernel" if ws else f"conv3x3_wgmma_kernel<CoutP={_cout_pad(Cout)}"
        if not kern.startswith(want):
            self._fail(f"{name}: kernel {kern}, expected {want}")
        if worst > 1.0:
            self._fail(f"{name} ({op}, N={N} Cin={Cin} Cout={Cout} {H}x{W} d={dil} s={stride}): err/bound {worst:.3g}")
        self.rows.append(dict(op=op, name=name, kernel=kern, N=N, Cin=Cin, Cout=Cout, H=H, W=W, dil=dil, stride=stride,
                              ws=ws, err_q=worst_q, ratio=worst, tags=tags, split_out="split" in tags))

    def conv3x3_slices(self, *args, **kw):
        a = self._bind("conv3x3_slices", args, kw)
        buf_in, buf_out = a["buf_in"], a["buf_out"]
        c_in0, Cin, c_out0, Cout = a["c_in0"], a["Cin"], a["c_out0"], a["Cout"]
        N, _, H, W = buf_in.shape
        d2s, lp, dil, stride = a["depth_to_space"], a["linear_prefix"], a["dilation"], a["stride"]
        ws = int(_lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, int(stride), int(dil)))
        before = buf_out.detach().clone()
        self.orig["conv3x3_slices"](*args, **kw)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        region = buf_out[:, c_out0:c_out0 + (Cout // 4 if d2s else Cout)]
        if not _outside_unchanged(buf_out, before, region):
            self._fail(f"conv3x3_slices wrote outside channels [{c_out0}, {c_out0 + Cout}) of its output buffer")
        del before
        tags = ["fp32"] + (["d2s"] if d2s else []) + (["lin"] if lp else []) + (["dil>=4"] if dil >= 4 else [])
        self._check_conv("conv3x3_slices", a["packed"], a["bias"], Cout, a["leaky_slope"], dil, stride, d2s, lp,
                         lambda n: buf_in[n:n + 1, c_in0:c_in0 + Cin].detach().double(),
                         lambda n: region[n:n + 1].detach(), N, Cin, H, W, ws, kern, tags)

    def conv3x3_split(self, *args, **kw):
        a = self._bind("conv3x3_split", args, kw)
        x, out, out_split = a["x"], a["out"], a["out_split"]
        c_in0, Cin, Cout, dil, lp, d2s = a["c_in0"], a["Cin"], a["Cout"], a["dilation"], a["linear_prefix"], \
            a["depth_to_space"]
        N, _, H, W = x.shape
        ws = int(_lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, 1, int(dil)))
        before = out_split.buf.clone() if out_split is not None else None
        self.orig["conv3x3_split"](*args, **kw)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        if out_split is not None:
            c0 = a["out_c0"]
            if not _groups_unchanged(out_split.buf, before, c0 // 8, (c0 + Cout - lp) // 8):
                self._fail(f"conv3x3_split wrote outside channels [{c0}, {c0 + Cout - lp}) of its split output")
            if not _pad_is_zero(out_split):
                self._fail("conv3x3_split: pad channels of the split output are not zero")
            del before

            def got_of(n):
                v = _split_values(out_split, n, c0, c0 + Cout - lp)
                return torch.cat([out[n:n + 1].double(), v], dim=1) if lp else v
        else:
            def got_of(n):
                return out[n:n + 1]
        tags = (["split"] if out_split is not None else []) + (["d2s"] if d2s else []) + (["lin"] if lp else []) + \
            (["dil>=4"] if dil >= 4 else [])
        self._check_conv("conv3x3_split", a["packed"], a["bias"], Cout, a["leaky_slope"], dil, 1, d2s, lp,
                         lambda n: _split_values(x, n, c_in0, c_in0 + Cin), got_of, N, Cin, H, W, ws, kern, tags,
                         lp if out_split is not None else None)

    def split_pack(self, act, src, c0):
        N, C, H, W = src.shape
        before = act.buf.clone()
        self.orig["pack"](act, src, c0)
        torch.cuda.synchronize()
        ok = _groups_unchanged(act.buf, before, c0 // 8, (c0 + C + 15) // 16 * 2) and _pad_is_zero(act)
        del before
        for n in range(N):
            one = ops.SplitAct.__new__(ops.SplitAct)
            one.channels, one.buf = act.channels, act.buf[n:n + 1]
            hi, lo = one.hi_lo()
            s = src[n:n + 1].detach()
            want_hi = s.bfloat16().float()
            ok = ok and torch.equal(hi[:, c0:c0 + C], want_hi) and torch.equal(lo[:, c0:c0 + C], (s - want_hi).bfloat16().float())
        if not ok:
            self._fail(f"SplitAct.pack of {C} channels at {c0} ({N}x{H}x{W}) is not the exact hi/lo split in place")
        self.rows.append(dict(op="SplitAct.pack", name=f"[{c0}:{c0 + C}]", kernel="split_pack", N=N, Cin=C, Cout=C, H=H,
                              W=W, dil=0, stride=1, ws=0, err_q=0.0, ratio=0.0 if ok else float("inf"), tags=[],
                              split_out=True))

    # ---- correlation ------------------------------------------------------------------------------------------
    def correlation(self, *args, **kw):
        a = self._bind("correlation", args, kw)
        d1, d2, out, md, slope = a["data1"], a["data2"], a["out"], a["max_displacement"], a["leaky_slope"]
        assert (a["pad_size"], a["kernel_size"], a["stride1"], a["stride2"], a["is_multiply"]) == (md, 1, 1, 1, 1)
        base = out._base if out is not None and out._base is not None else out
        before = base.clone() if base is not None else None
        res = self.orig["correlation"](*args, **kw)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        if base is not None and not _outside_unchanged(base, before, out):
            self._fail("correlation wrote outside its slot of the concat buffer")
        del before
        N, C, H, W = d1.shape
        D = (2 * md + 1) ** 2
        sl = channel_slopes(D, slope, 0, d1.device)
        worst, worst_q = 0.0, 0.0
        with torch.no_grad():
            for n in range(N):
                f1, f2 = d1[n:n + 1].detach().double(), d2[n:n + 1].detach().double()
                pre = torch_ref.correlation(f1, f2, md)
                Q = (torch_ref.correlation(f1 * f1, f2 * f2, md) * C).sqrt() / C
                S = torch_ref.correlation(f1.abs(), f2.abs(), md)
                r, rq = judge(res[n:n + 1], pre, sl, EPS_Q * Q + EPS_S * S, Q)
                worst, worst_q = max(worst, r), max(worst_q, rq)
        if worst > 1.0:
            self._fail(f"correlation N={N} C={C} {H}x{W} md={md} ({kern}): err/bound {worst:.3g}")
        self.rows.append(dict(op="correlation", name=f"md={md}", kernel=kern, N=N, Cin=C, Cout=D, H=H, W=W, dil=0,
                              stride=1, ws=0, err_q=worst_q, ratio=worst, tags=[], split_out=False))
        return res

    # ---- fused warp -------------------------------------------------------------------------------------------
    def _upsample_ratio(self, got, coarse, f, scale=1.0):
        """Exact-fp32 check of Upsample(f) (times scale) against float64."""
        c = coarse.detach().double()
        ref = torch_ref.upsample(c, f) * scale
        S = torch_ref.upsample(c.abs(), f) * abs(scale)
        return float(_ratio((got.double() - ref).abs(), EPS_S * S).max())

    def warp_mask(self, *args, **kw):
        a = self._bind("warp_mask", args, kw)
        res = self.orig["warp_mask"](*args, **kw)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        out, fup, mup = res
        x, fc, mc, w, b, t = (a[k] for k in ("x", "flow_coarse", "mask_coarse", "weight", "bias", "tradeoff"))
        up, scale, stride, slope, border = a["upsample"], a["scale"], a["stride"], a["leaky_slope"], a["border_mode"]
        N, C, H, W = x.shape
        F = w.shape[0]
        exact = kern.startswith("deform_fwd_kernel")          # the SIMT kernel of the training graph
        # warp_mma_kernel (below 4 px, F <= 128) gathers tap by tap at the SIMT kernel's positions: its offsets are
        # fl(fl(f * scale) / stride) from the up-sampled flow it also returns, its positions fl((y - 1 + i) + d), so the
        # reference's positions are its own.  Each bilinear sample is formed in fp32 (corner weights (1 - l) * (1 - l'),
        # four products, three sums: <= 6u of sum |w_corner v_corner|, inside 2^-20 S), then split into bf16 hi + lo
        # and multiplied hi*hi + hi*lo + lo*hi into fp32 accumulators, as the wgmma convolution does: the tensor-core
        # bound holds with no position term.
        through_linearity = not exact and not kern.startswith("warp_mma_kernel")
        eps_q = 0.0 if exact else EPS_Q
        sl = channel_slopes(F, slope, 0, x.device)
        worst = worst_q = worst_up = worst_fixed = 0.0
        with torch.no_grad():
            wd = w.detach().double()
            ys = torch.arange(H, dtype=torch.float64, device=x.device).view(1, 1, H, 1)
            xs = torch.arange(W, dtype=torch.float64, device=x.device).view(1, 1, 1, W)
            for n in range(N):
                worst_up = max(worst_up, self._upsample_ratio(fup[n:n + 1], fc[n:n + 1], up))
                if mc is not None:
                    worst_up = max(worst_up, self._upsample_ratio(mup[n:n + 1], mc[n:n + 1], up))
                xn, fn = x[n:n + 1].detach().double(), fup[n:n + 1].detach()
                conv = _warp_conv(xn, fn, wd, scale, stride, border)
                Q = _warp_conv(xn * xn, fn, wd * wd, scale, stride, border).sqrt()
                S = _warp_conv(xn.abs(), fn, wd.abs(), scale, stride, border)
                bb = b.detach().double().view(1, -1, 1, 1) if b is not None else 0.0
                pre, S = conv + bb, S + (b.detach().double().abs().view(1, -1, 1, 1) if b is not None else 0.0)
                sig = torch.sigmoid(mup[n:n + 1].detach().double()) if mc is not None else 1.0
                pre, Q, S = pre * sig, Q * sig, S * sig
                if t is not None:
                    tn = t[n:n + 1].detach().double()
                    pre, S = pre + tn, S + tn.abs()
                bound = eps_q * Q + EPS_S * S
                worst_fixed = max(worst_fixed, judge(out[n:n + 1], pre, sl, bound, Q)[0])
                if through_linearity:
                    # through linearity every tap row samples the zero-corner operator at the one rounded position
                    # fl(y + d) shifted by whole pixels, and the MXNet-1.5 band correction at fl((y - 1 + i) + d), the
                    # tap-by-tap operator's positions: each part is off by up to one ulp of |y| + |d| + 1 (likewise
                    # columns), and the correction is the difference of the two rules
                    dy, dx = (d.unsqueeze(1).abs() for d in _warp_offsets(fn, scale, stride))
                    dev_y, dev_x = 2.0 ** -22 * (ys + dy + 2), 2.0 ** -22 * (xs + dx + 2)
                    for rule, k in ((ops.BORDER_ZERO_CORNER, 1 if border == ops.BORDER_ZERO_CORNER else 2),
                                    (border, 0 if border == ops.BORDER_ZERO_CORNER else 1)):
                        if k:
                            bound = bound + k * _position_term(
                                lambda sy, sx: _warp_conv(xn, fn, wd, scale, stride, rule, sy, sx) * sig, dev_y, dev_x)
                r, rq = judge(out[n:n + 1], pre, sl, bound, Q)
                if r > 1.0:
                    e = (out[n:n + 1].double() - activate(pre, sl)).abs()
                    i = int(torch.argmax(_ratio(e, bound)))
                    f_, y_, x_ = i // (H * W), (i // W) % H, i % W
                    d0, d1 = (float(d[0, y_, x_]) for d in _warp_offsets(fn, scale, stride))
                    self._fail(f"  worst element n={n} f={f_} y={y_} x={x_}: got {float(out[n, f_, y_, x_]):.9g} ref "
                               f"{float(activate(pre, sl)[0, f_, y_, x_]):.9g} Q {float(Q[0, f_, y_, x_]):.3g} S "
                               f"{float(S[0, f_, y_, x_]):.3g} bound {float(bound[0, f_, y_, x_]):.3g}; offsets ({d0:.9g}, {d1:.9g})")
                worst, worst_q = max(worst, r), max(worst_q, rq)
        if max(worst, worst_up) > 1.0:
            self._fail(f"warp_mask N={N} C={C} F={F} {H}x{W} up={up} ({kern}): err/bound {worst:.3g} "
                       f"({worst_fixed:.3g} without the position term), flow/mask upsample {worst_up:.3g}")
        self.rows.append(dict(op="warp_mask", name=f"stride={stride:g} ({worst_fixed:.3f})", kernel=kern, N=N, Cin=C,
                              Cout=F, H=H, W=W, dil=0, stride=1, ws=0, err_q=worst_q, ratio=max(worst, worst_up), tags=[],
                              split_out=False))
        return res

    # ---- upsample, cascade input ------------------------------------------------------------------------------
    def upsample(self, *args, **kw):
        a = self._bind("upsample", args, kw)
        res = self.orig["upsample"](*args, **kw)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        x, f, scale = a["x"], a["factor"], a["scale"]
        with torch.no_grad():
            worst = max(self._upsample_ratio(res[n:n + 1], x[n:n + 1], f, scale) for n in range(x.shape[0]))
        if worst > 1.0:
            self._fail(f"upsample x{f} of {tuple(x.shape)}: err/bound {worst:.3g}")
        N, C, H, W = x.shape
        self.rows.append(dict(op="upsample", name=f"x{f}", kernel=kern, N=N, Cin=C, Cout=C, H=H, W=W, dil=0, stride=1,
                              ws=0, err_q=0.0, ratio=worst, tags=[], split_out=False))
        return res

    def image_warp_concat(self, *args, **kw):
        a = self._bind("image_warp_concat", args, kw)
        c30, c40 = res = self.orig["image_warp_concat"](*args, **kw)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        im1, im2, fq, mq, scale = a["im1"], a["im2"], a["flow_q"], a["mask_q"], a["scale"]
        N, Ci, H, W = im2.shape
        ok = c30 is None or torch.equal(c30, torch.cat([im1, torch.zeros_like(im1[:, :1])], dim=1))
        worst = 0.0
        with torch.no_grad():
            ys = torch.arange(H, dtype=torch.float64, device=im2.device).view(1, 1, H, 1)
            xs = torch.arange(W, dtype=torch.float64, device=im2.device).view(1, 1, 1, W)
            for n in range(N):
                i2 = im2[n:n + 1].double()
                disp = torch_ref.upsample(fq[n:n + 1].double(), 4) * scale          # (y, x)
                warped = torch_ref.reconstruction2d(i2, disp)
                S = torch_ref.reconstruction2d(i2.abs(), disp)
                # the kernel's sample position p + d is rounded in fp32 after an fp32 Upsample(4) of the flow
                shift = lambda sy, sx: torch_ref.reconstruction2d(  # noqa: E731
                    i2, disp + torch.tensor([sy, sx], dtype=torch.float64, device=i2.device).view(1, 2, 1, 1))
                bound = EPS_S * S + _position_term(shift, EPS_S * (ys + disp[:, :1].abs() + 1),
                                                   EPS_S * (xs + disp[:, 1:].abs() + 1))
                worst = max(worst, float(_ratio((c40[n:n + 1, :Ci].double() - warped).abs(), bound).max()))
                m = torch_ref.upsample(mq[n:n + 1].double(), 4)
                merr = (c40[n:n + 1, Ci:].double() - (torch.sigmoid(m) - 0.5)).abs()
                worst = max(worst, float(_ratio(merr, EPS_S * (1 + m.abs())).max()))
        if not ok or worst > 1.0:
            self._fail(f"image_warp_concat {N}x{Ci}x{H}x{W}: c30 exact {ok}, c40 err/bound {worst:.3g}")
        self.rows.append(dict(op="image_warp_concat", name="c30/c40", kernel=kern, N=N, Cin=Ci, Cout=Ci + 1, H=H, W=W,
                              dil=0, stride=1, ws=0, err_q=0.0, ratio=worst if ok else float("inf"), tags=[],
                              split_out=False))
        return res

    # ---- report -----------------------------------------------------------------------------------------------
    def report(self):
        for r in self.rows:
            plan = f"ws={r['ws']}" if r["ws"] else "-"
            print(f"{self.run:8s} {r['op']:17s} {r['name']:24s} {r['kernel']:42s} N={r['N']} {r['Cin']}->{r['Cout']} "
                  f"{r['H']}x{r['W']} d={r['dil']} s={r['stride']} {plan:12s} err/Q={r['err_q']:.2e} "
                  f"err/bound={r['ratio']:.3f}")
        for tag, (name, rs) in sorted(self.controls.items()):
            print(f"{self.run:8s} control {tag:7s} on {name}: bf16-only err/bound={rs['bf16']:.3g}, "
                  f"dropped tap err/bound={rs['tap']:.3g}")


def _named_model(cls):
    m = cls()
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(named_init(k.replace("MaskFlownet_S.", "") if cls is network.MaskFlownetS else k, p.shape))
    return m.cuda()


def _images_u8(seed, n, h, w):
    out = []
    for t in seeded_images(seed=seed, n=n, h=h, w=w):
        lo, hi = t.amin(), t.amax()
        out.append(((t - lo) / (hi - lo) * 255).round().to(torch.uint8).contiguous().cuda())
    return out


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


RUNS = {   # run: (model class, batch, H, W, image seed) -- bench.py's configs[1], [3], [4] (padded frame) and [2]
    "fwd": (network.MaskFlownetS, 8, 448, 1024, 21),
    "cascade": (network.MaskFlownet, 4, 448, 1024, 22),
    "odd": (network.MaskFlownetS, 4, 576, 960, 23),
    "train": (network.MaskFlownetS, 8, 384, 512, 24),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
def test_every_launch_of_the_benchmarked_forward_against_float64(run, monkeypatch):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cls, N, H, W, seed = RUNS[run]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    rec = Recorder(monkeypatch, run)         # before the model packs anything
    model = _named_model(cls)
    u1, u2 = _images_u8(seed=seed, n=N, h=H, w=W)
    if run == "train":
        model.train()
        a, b, _ = network.centralize(u1.float() / 255.0, u2.float() / 255.0)
        with torch.enable_grad():
            preds = model(a, b)[0]
        assert preds[-1].requires_grad
    else:
        model.eval()
        flow = network.predict_flow(model, u1, u2)
        assert flow.shape == (N, 2, H, W) and bool(torch.isfinite(flow).all())
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    rec.report()
    print(f"{run}: {len(rec.rows)} launches checked in {secs:.1f} s, peak {peak:.2f} GiB allocated")
    assert not rec.failures, "\n".join(rec.failures)

    # coverage: this run checked what the benchmark runs
    convs = [r for r in rec.rows if r["op"] in ("conv3x3_slices", "conv3x3_split")]
    assert len(convs) == _expected_convs(run), (len(convs), _expected_convs(run))
    print(f"{run}: kernel variants {sorted({r['kernel'] for r in convs})}")
    want_kinds = {"fp32", "dil>=4"} if run == "train" else set(Recorder.KINDS)
    assert set(rec.controls) == want_kinds, sorted(rec.controls)
    for tag, (name, rs) in rec.controls.items():
        assert min(rs.values()) >= CONTROL_MARGIN, (tag, name, rs)
    if run != "train":
        tma_dils = {r["dil"] for r in convs if r["op"] == "conv3x3_split"}
        assert {1, 2, 4, 8, 16} <= tma_dils, tma_dils
    if run == "cascade":
        assert any(r["split_out"] and r["ws"] > 0 and r["N"] == 4 and r["H"] == 112 for r in convs), \
            "no split-K launch with split output at level 2"
        assert any(r["op"] == "warp_mask" and r["kernel"] == "warp_lin_kernel" and r["Cout"] == 196 for r in rec.rows)
