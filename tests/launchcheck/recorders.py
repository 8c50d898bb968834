"""The recorders: each wraps the `ops` functions a graph calls, runs the original, synchronises and checks that launch
against float64 as it happens.  Recorder: the forward; BackwardRecorder: the training step's backward; ServingRecorder:
the serving shapes; BF16Recorder: the bf16 inference mode."""
import inspect
import math

import numpy as np
import torch
import torch.nn.functional as tF

from maskflownet_b200 import _lib, losses, network, ops
from oracle import torch_ref

from .backward import (EPS_WIRING, TAPS, U, _f32, _tap_positions, corner_scatter, corr_bwd_ref, epe_backward_bounds,
                       epe_forward_bound, epe_q_controls, gamma, image_warp_flow_slopes, judge_bound, sigmoid_error,
                       upsample_T, warp_bwd_S, warp_bwd_ref)
from .bounds import (EPS_Q, EPS_S, _bf, _bf16_pad_is_zero, _cout_pad, _groups_unchanged, _outside_unchanged,
                     _pad_is_zero, _position_term, _ratio, _split_values, _warp_conv, _warp_offsets, activate,
                     bf16_bound, bf16_near_misses, bf16_terms, channel_slopes, conv_near_misses, conv_terms, judge,
                     split_storage_term)


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


def _corr_replicate(f1, f2, md):
    """torch_ref.correlation with f2 padded by replicating its border instead of by zeros (a near miss)."""
    H, W = f1.shape[2:]
    p = tF.pad(f2, (md,) * 4, mode="replicate")
    return torch.stack([(f1 * p[:, :, md + dy:md + dy + H, md + dx:md + dx + W]).sum(dim=1) / f1.shape[1]
                        for dy in range(-md, md + 1) for dx in range(-md, md + 1)], dim=1)


def _row(op, name, kernel, shape, ratio, **kw):
    N, C, H, W = shape
    r = dict(op=op, name=name, kernel=kernel, N=N, Cin=C, Cout=C, H=H, W=W, dil=0, stride=1, ws=0, err_q=0.0,
             ratio=ratio, tags=[], split_out=False, split_all=False)
    r.update(kw)
    return r


class ServingRecorder(Recorder):
    """Recorder plus: where each launch's split-K plan splits every tile, the controls of test_serving_shapes.py
    (self.extra: tag -> (layer, err/bound)) and the warp_mma_kernel controls (in self.controls, the base's format), and
    ops.preprocess / ops.postprocess against oracle/prepost_ref."""

    def __init__(self, monkeypatch, run):
        super().__init__(monkeypatch, run)
        self.extra = {}
        for name in ("preprocess", "postprocess"):
            self.orig[name] = getattr(ops, name)
            monkeypatch.setattr(ops, name, getattr(self, name))

    # ---- convolutions ---------------------------------------------------------------------------------------------
    def _check_conv(self, op, packed, bias, Cout, slope, dil, stride, d2s, lp, x_of, got_of, N, Cin, H, W, ws, kern,
                    tags, store_from=None):
        OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
        # the base controls drop tap (0, 0): they say something only where that tap reads inside the image for some
        # output pixel, so launches where it never does (1x1 levels) leave them to a later launch of the same kind
        reach = (OH - 1) * stride >= dil and (OW - 1) * stride >= dil
        super()._check_conv(op, packed, bias, Cout, slope, dil, stride, d2s, lp, x_of, got_of, N, Cin, H, W, ws, kern,
                            tags if reach else [], store_from)
        row = self.rows[-1]
        row["tags"], row["split_out"] = tags, "split" in tags
        row["split_all"] = ws > 0 and ws % (4 * N * Cout * OH * OW) == 0     # the workspace holds k whole outputs
        want = []
        # (on an image wider and taller than 4 px: below that the correlation's last channels, the last chunk of the
        # first dense-block layer, lie wholly outside and are zero)
        if op == "conv3x3_split" and row["split_all"] and not d2s and Cin > 16 and min(H, W) > 4 and \
                "chunk" not in self.extra:
            want.append("chunk")
        if not d2s and dil > 1 and dil >= max(H, W) and "pad" not in self.extra:
            want.append("pad")
        if want:
            self._conv_controls(want, packed, bias, Cout, slope, dil, stride, lp, x_of(0), store_from)

    def _conv_controls(self, tags, packed, bias, Cout, slope, dil, stride, lp, x, store_from):
        w = self.packs[packed.data_ptr()][0].double()
        b = bias.detach().double().view(1, -1, 1, 1) if bias is not None else None
        name = self.names.get(packed.data_ptr(), "?")
        sl = channel_slopes(Cout, slope, lp, w.device)
        with torch.no_grad():
            pre, Q, S = conv_terms(x, w, b.view(-1) if b is not None else None, stride, dil)
            bound = EPS_Q * Q + EPS_S * S + split_storage_term(pre, store_from)
            for tag in tags:
                if tag == "chunk":      # the input channels of the last 16-channel chunk dropped
                    wd = w.clone()
                    wd[:, (w.shape[1] - 1) // 16 * 16:] = 0
                    alt = tF.conv2d(x, wd, stride=stride, padding=dil, dilation=dil)
                else:                   # the padding replicates the border instead of reading zeros
                    alt = tF.conv2d(tF.pad(x, (dil,) * 4, mode="replicate"), w, stride=stride, dilation=dil)
                if b is not None:
                    alt = alt + b
                self.extra[tag] = (name, judge(activate(alt, sl), pre, sl, bound, Q)[0])

    # ---- correlation: replicate padding at 1x1 --------------------------------------------------------------------
    def correlation(self, *args, **kw):
        res = super().correlation(*args, **kw)
        a = self._bind("correlation", args, kw)
        d1, d2, md, slope = a["data1"], a["data2"], a["max_displacement"], a["leaky_slope"]
        N, C, H, W = d1.shape
        if (H, W) == (1, 1) and "corr_pad" not in self.extra:
            with torch.no_grad():
                f1, f2 = d1[:1].detach().double(), d2[:1].detach().double()
                pre = torch_ref.correlation(f1, f2, md)
                Q = (torch_ref.correlation(f1 * f1, f2 * f2, md) * C).sqrt() / C
                S = torch_ref.correlation(f1.abs(), f2.abs(), md)
                sl = channel_slopes(pre.shape[1], slope, 0, d1.device)
                r = judge(activate(_corr_replicate(f1, f2, md), sl), pre, sl, EPS_Q * Q + EPS_S * S, Q)[0]
            self.extra["corr_pad"] = (f"correlation md={md} C={C} 1x1", r)
        return res

    # ---- warp: the warp_mma_kernel controls -----------------------------------------------------------------------
    def warp_mask(self, *args, **kw):
        res = super().warp_mask(*args, **kw)
        if self.rows[-1]["kernel"].startswith("warp_mma_kernel") and "warp_mma" not in self.controls:
            a = self._bind("warp_mask", args, kw)
            _, fup, mup = res
            x, fc, mc, w, b, t = (a[k] for k in ("x", "flow_coarse", "mask_coarse", "weight", "bias", "tradeoff"))
            scale, stride, border = a["scale"], a["stride"], a["border_mode"]
            with torch.no_grad():
                xn, fn, wd = x[:1].detach().double(), fup[:1].detach(), w.detach().double()
                sig = torch.sigmoid(mup[:1].detach().double()) if mc is not None else 1.0
                bb = b.detach().double().view(1, -1, 1, 1) if b is not None else 0.0
                tn = t[:1].detach().double() if t is not None else 0.0

                def pre_of(xx, ww):
                    return (_warp_conv(xx, fn, ww, scale, stride, border) + bb) * sig + tn
                pre = pre_of(xn, wd)
                Q = _warp_conv(xn * xn, fn, wd * wd, scale, stride, border).sqrt() * sig
                S = (_warp_conv(xn.abs(), fn, wd.abs(), scale, stride, border) +
                     (b.detach().double().abs().view(1, -1, 1, 1) if b is not None else 0.0)) * sig
                S = S + (tn.abs() if t is not None else 0.0)
                bound = EPS_Q * Q + EPS_S * S
                sl = channel_slopes(w.shape[0], a["leaky_slope"], 0, x.device)
                bf = lambda v: v.to(torch.bfloat16).double()  # noqa: E731
                w_drop = wd.clone()
                w_drop[:, :, 1, 1] = 0      # the centre tap: at 2x2 the corner taps may all fall outside
                self.controls["warp_mma"] = (
                    f"warp_mask {x.shape[2]}x{x.shape[3]} F={w.shape[0]}",
                    {"bf16": judge(activate(pre_of(bf(xn), bf(wd)), sl), pre, sl, bound, Q)[0],
                     "tap": judge(activate(pre_of(xn, w_drop), sl), pre, sl, bound, Q)[0]})
        return res

    # ---- pre / post-processing against the oracle (tolerances of test_ops_gpu's oracle test) ----------------------
    def preprocess(self, img1, img2, out_hw=None):
        from oracle import prepost_ref
        res = self.orig["preprocess"](img1, img2, out_hw)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        ra, rb, rm = prepost_ref.preprocess(img1.cpu().numpy(), img2.cpu().numpy(), out_hw)
        o1, o2, m = (t.cpu().numpy() for t in res)
        r = max(np.abs(m - rm).max() / 2e-6, np.abs(o1 - ra).max() / 1e-5, np.abs(o2 - rb).max() / 1e-5)
        if r > 1.0:
            self._fail(f"preprocess {tuple(img1.shape)} -> {out_hw}: err/tolerance {r:.3g}")
        self.rows.append(_row("preprocess", f"-> {o1.shape[2]}x{o1.shape[3]}", kern, tuple(img1.shape), float(r)))
        return res

    def postprocess(self, pred, H, W, flip_channels=True, is_flow=True):
        from oracle import prepost_ref
        res = self.orig["postprocess"](pred, H, W, flip_channels, is_flow)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        ref = prepost_ref.postprocess(pred.detach().cpu().numpy(), H, W, flip_channels, is_flow)
        r = float(np.abs(res.cpu().numpy() - ref).max()) / (1e-4 if is_flow else 1e-5)
        if r > 1.0:
            self._fail(f"postprocess {tuple(pred.shape)} -> {H}x{W} (flow {is_flow}): err/tolerance {r:.3g}")
        self.rows.append(_row("postprocess", "flow" if is_flow else "mask", kern, tuple(pred.shape), r, H=H, W=W))
        return res

    def report(self):
        super().report()
        for tag, (name, r) in sorted(self.extra.items()):
            print(f"{self.run:8s} control {tag:8s} on {name}: err/bound={r:.3g}")
        worst = {}
        for r in self.rows:
            key = (r["op"], r["kernel"].split("<")[0])
            worst[key] = max(worst.get(key, 0.0), r["ratio"])
        for (op, kern), v in sorted(worst.items()):
            print(f"{self.run:8s} worst {op:17s} {kern:30s} err/bound={v:.3f}")


def _cover_tiny(rec, convs):
    warps = {(r["H"], r["W"], r["kernel"]) for r in rec.rows if r["op"] == "warp_mask"}
    assert (2, 2, "warp_mma_kernel") in warps, warps                      # level 5
    assert (4, 4, "warp_lin_kernel") in warps, warps                      # level 4, the through-linearity minimum
    corr = {(r["H"], r["Cin"]): r["kernel"] for r in rec.rows if r["op"] == "correlation"}
    assert (1, 196) in corr and (2, 128) in corr, corr
    assert {c for (_, c), k in corr.items() if k.startswith("corr_rb_kernel")} == {196, 128, 96, 64}, corr
    assert any(r["op"] == "conv3x3_split" and r["dil"] == 16 and (r["H"], r["W"]) == (16, 16) for r in convs)
    split_levels = {r["H"] for r in convs if r["op"] == "conv3x3_split" and r["split_all"]}
    assert {1, 2, 4, 8, 16} <= split_levels, split_levels                 # a reduce launch at every decoder level
    assert {"chunk", "pad", "corr_pad"} <= set(rec.extra) and "warp_mma" in rec.controls


def _cover_tiny_cascade(rec, convs):
    assert any(r["op"] == "warp_mask" and r["kernel"].startswith("deform_fwd_kernel") and r["Cout"] == 196 and
               (r["H"], r["W"]) == (1, 1) for r in rec.rows)
    assert any(r["op"] == "correlation" and r["name"] == "md=2" and (r["H"], r["W"]) == (1, 1) for r in rec.rows)
    assert any(r["op"] == "image_warp_concat" and (r["H"], r["W"]) == (64, 64) for r in rec.rows)
    assert "warp_mma" in rec.controls and "corr_pad" in rec.extra


class BF16Recorder(Recorder):
    """Recorder with the bf16 bound: every convolution must have run the one-product variant."""

    KINDS = ("fp32-s2", "bf16-io", "d2s", "lin", "dil>=4", "split-k")

    def _check_conv(self, op, packed, bias, Cout, slope, dil, stride, d2s, lp, x_of, got_of, N, Cin, H, W, ws, kern,
                    tags, store_from=None, x_full_of=None):
        w_full, transposed = self.packs[packed.data_ptr()]
        name = self.names.get(packed.data_ptr(), "?")
        assert transposed == d2s, name
        w_full = w_full.double()
        w = w_full.float().bfloat16().double()
        b = bias.detach().double() if bias is not None else None
        F = Cout // 4 if d2s else Cout
        sl = channel_slopes(F, slope, lp, w.device)
        worst = 0.0
        if ws:
            tags = tags + ["split-k"]
        with torch.no_grad():
            for n in range(N):
                x = x_of(n)
                pre, S = bf16_terms(x, w, b, stride, dil, transposed)
                bound = bf16_bound(pre, S, store_from)
                worst = max(worst, judge(got_of(n), pre, sl, bound, S)[0])
                for tag in tags:
                    if tag not in self.controls:
                        xf = x_full_of(n) if x_full_of is not None else x
                        self.controls[tag] = (name, {k: judge(activate(v, sl), pre, sl, bound, S)[0] for k, v in
                                                     bf16_near_misses(xf, w_full, x, w, b, stride, dil, transposed).items()})
                del x, pre, S, bound
        if ws:
            ok = kern == "conv3x3_wgmma_reduce_kernel<bf16>"
        else:
            ok = kern.startswith(f"conv3x3_wgmma_kernel<CoutP={_cout_pad(Cout)}") and kern.endswith(",bf16>")
        if not ok:
            self._fail(f"{name}: kernel {kern}, expected the one-product (bf16) variant")
        if worst > 1.0:
            self._fail(f"{name} ({op}, N={N} Cin={Cin} Cout={Cout} {H}x{W} d={dil} s={stride}): err/bound {worst:.3g}")
        self.rows.append(dict(op=op, name=name, kernel=kern, N=N, Cin=Cin, Cout=Cout, H=H, W=W, dil=dil, stride=stride,
                              ws=ws, err_q=0.0, ratio=worst, tags=tags, split_out=store_from is not None))

    def conv3x3_slices(self, *args, **kw):
        a = self._bind("conv3x3_slices", args, kw)
        if not a["bf16"]:
            self._fail("conv3x3_slices ran without bf16 in a bf16 forward")
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
        tags = (["fp32-s2"] if stride == 2 else []) + (["dil>=4"] if dil >= 4 else [])
        self._check_conv("conv3x3_slices", a["packed"], a["bias"], Cout, a["leaky_slope"], dil, stride, d2s, lp,
                         lambda n: _bf(buf_in[n:n + 1, c_in0:c_in0 + Cin].detach()),
                         lambda n: region[n:n + 1].detach(), N, Cin, H, W, ws, kern, tags,
                         x_full_of=lambda n: buf_in[n:n + 1, c_in0:c_in0 + Cin].detach().double())

    def conv3x3_split(self, *args, **kw):
        a = self._bind("conv3x3_split", args, kw)
        x, out, out_split = a["x"], a["out"], a["out_split"]
        if not (a["bf16"] and x.bf16 and (out_split is None or out_split.bf16)):
            self._fail("conv3x3_split ran without bf16 operands in a bf16 forward")
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
                self._fail(f"conv3x3_split wrote outside channels [{c0}, {c0 + Cout - lp}) of its bf16 output")
            if not _bf16_pad_is_zero(out_split):
                self._fail("conv3x3_split: pad channels of the bf16 output are not zero")
            del before

            def got_of(n):
                v = _split_values(out_split, n, c0, c0 + Cout - lp)
                return torch.cat([out[n:n + 1].double(), v], dim=1) if lp else v
        else:
            def got_of(n):
                return out[n:n + 1]
        tags = (["bf16-io"] if out_split is not None else []) + (["d2s"] if d2s else []) + (["lin"] if lp else []) + \
            (["dil>=4"] if dil >= 4 else [])
        self._check_conv("conv3x3_split", a["packed"], a["bias"], Cout, a["leaky_slope"], dil, 1, d2s, lp,
                         lambda n: _split_values(x, n, c_in0, c_in0 + Cin), got_of, N, Cin, H, W, ws, kern, tags,
                         lp if out_split is not None else None)

    def split_pack(self, act, src, c0):
        if not act.bf16:
            self._fail("SplitAct.pack into a split activation in a bf16 forward")
            return self.orig["pack"](act, src, c0)
        N, C, H, W = src.shape
        before = act.buf.clone()
        self.orig["pack"](act, src, c0)
        torch.cuda.synchronize()
        ok = _groups_unchanged(act.buf, before, c0 // 8, (c0 + C + 15) // 16 * 2) and _bf16_pad_is_zero(act)
        del before
        hi, lo = act.hi_lo()
        ok = ok and torch.equal(hi[:, c0:c0 + C], src.detach().bfloat16().float()) and not bool(lo.any())
        if not ok:
            self._fail(f"SplitAct.pack of {C} channels at {c0} ({N}x{H}x{W}) is not the bf16 rounding in place")
        self.rows.append(dict(op="SplitAct.pack", name=f"[{c0}:{c0 + C}]", kernel="split_pack<bf16>", N=N, Cin=C,
                              Cout=C, H=H, W=W, dil=0, stride=1, ws=0, err_q=0.0, ratio=0.0 if ok else float("inf"),
                              tags=[], split_out=True))

    def report(self):
        for r in self.rows:
            plan = f"ws={r['ws']}" if r["ws"] else "-"
            print(f"{self.run:8s} {r['op']:17s} {r['name']:24s} {r['kernel']:42s} N={r['N']} {r['Cin']}->{r['Cout']} "
                  f"{r['H']}x{r['W']} d={r['dil']} s={r['stride']} {plan:12s} err/bound={r['ratio']:.3f}")
        for tag, (name, rs) in sorted(self.controls.items()):
            print(f"{self.run:8s} control {tag:8s} on {name}: fp32-accurate err/bound={rs['fp32']:.3g}, "
                  f"dropped tap err/bound={rs['tap']:.3g}")

    # the fp32 operators of a bf16 forward run unchecked here (their own tests check them)
    def correlation(self, *args, **kw):
        return self.orig["correlation"](*args, **kw)

    def warp_mask(self, *args, **kw):
        return self.orig["warp_mask"](*args, **kw)

    def upsample(self, *args, **kw):
        return self.orig["upsample"](*args, **kw)

    def image_warp_concat(self, *args, **kw):
        return self.orig["image_warp_concat"](*args, **kw)
