"""Every launch of the unsupervised fine-tuning step against float64, the frame's edges included.

PipelineFlownet.train_batch_unsupervised runs the network at batch 2N on [a; b] -> [b; a], up-samples the last
prediction and calls losses.unsupervised_loss, whose launches the supervised step never runs: the forward-backward check
(mfn_flow_consistency), the stand-alone image warp ops.reconstruction2d (mfn_grid_generator_warp_forward +
mfn_bilinear_sampler_forward and their backwards) on full-resolution flows, and the census and smoothness Functions.
This file builds that step and checks every launch while it happens: the network, ops.upsample and its backward through
Recorder and BackwardRecorder of launchcheck.recorders, the launches above through the wrappers below.
Each wrapper runs the original, synchronises, and judges that launch alone, on the values it read, against float64.

Bounds, per element (gamma_L = L u / (1 - L u), u = 2^-24, S the same sum on absolute values):
  * grid generator, forward: grid = fl(fl(fl(f + p) / s) - 1), s = (W - 1) / 2 exact in fp32 -> gamma_3 S with
    S = (|f| + p) / s + 1; backward: fl(g / s) -> gamma_1 |g / s|.
  * bilinear sampler, forward: the sampler reads the fp32 grid g and de-normalises it to fl(fl(g + 1) (W - 1)) / 2, two
    roundings of a product: within dv = gamma_2 |v| px of the exact v = (g + 1)(W - 1) / 2 (the halving is exact), and
    the same along y.  Corner weights wy * wx (1 rounding; each 1 - l is off by at most 2u absolutely), four
    products and sums (5): gamma_6 S + 4u sum |corners| + dh max |d/dh| + dv max |d/dv| + |Delta| dh dv, the slopes
    over every cell the fp32 position may lie in, with the zero padding's cliff (the whole pixel value, not a
    neighbour difference) where a corner leaves the frame.
  * bilinear sampler, position backward: the slope of the cell of the fp32 position, times (W - 1) / 2, judged by
    image_warp_flow_slopes (gamma_(C+6) S and the position terms; either cell where the position may lie on either side
    of an integer).  The data gradient is not requested: the images are data.
  * census and smoothness: census_bounds / smoothness_bounds of launchcheck.unsup_loss (there E plays S's part).  The
    smoothness gradient is judged with the signs of the second differences as the kernel evaluates them in fp32
    (kernel_signs): Upsample(4) makes most of them zero in exact arithmetic, where rounding decides the sign, and the
    float64 sign's allowance would be as large as the gradient itself, so that no control could fail it.
  * flow_consistency: the decisions against the float64 rule of launchcheck.bidirectional outside its ambiguous pixels.
Sensitivity (a control per new kind must fail by CONTROL_MARGIN on a real launch) and coverage (launch counts equal the
graph's; sampled corners leave the frame on all four sides; the occluded share lies strictly inside (0, 1)) are
asserted.  test_sampler_bounds_accept_kernel_arithmetic_and_reject_controls checks the same bounds on the CPU against
the kernels' arithmetic (the backward compiled from its source, the forwards' fp32 order in torch).

The network starts from the named weights of launchcheck.inputs with its flow heads (pred_flow*, dc_conv7) scaled by
FLOW_HEAD_SCALE: unscaled, the random heads give flows of several pixels that disagree between the two directions, so
that 99 % of the pixels fail the consistency check and the census sees almost nothing.  Scaled, the flows stay below
2 px, the size a fine-tuning run starting from a trained network sees on consecutive frames, and a fifth of the pixels
(a twentieth in the cascade) pass the check.
"""
import time

import numpy as np
import pytest
import torch

from maskflownet_b200 import losses, network, ops, pipeline
from oracle import unsup_ref

from launchcheck import fp64_references  # noqa: F401
from launchcheck.backward import _gather0, gamma, image_warp_flow_slopes, judge_bound, sampler_cell_slopes
from launchcheck.bidirectional import consistency_ref
from launchcheck.bounds import CONTROL_MARGIN, U, _ratio
from launchcheck.emu import build, ptr
from launchcheck.inputs import FLOW_HEAD_SCALE, _images_u8, _named_model
from launchcheck.recorders import BackwardRecorder, Recorder
from launchcheck.unsup_loss import census_backward_control, census_bounds, ratio as unsup_ratio, smoothness_bounds

GRIDGEN_L, GRIDGEN_BWD_L = 3, 1        # f + p, __fdiv_rn, - 1 / __fdiv_rn
SAMPLER_L = 6                          # wy * wx, then four products and sums
UPSAMPLE = 4                           # PipelineFlownet.scale: the last prediction is at a quarter of the resolution


# ------------------------------------------------------------------------------------------------------------------
# float64 references and bounds (any device)
# ------------------------------------------------------------------------------------------------------------------
def _pixels(N, H, W, dev):
    ys = torch.arange(H, dtype=torch.float64, device=dev).view(1, H, 1).expand(N, H, W)
    xs = torch.arange(W, dtype=torch.float64, device=dev).view(1, 1, W).expand(N, H, W)
    return ys, xs


def _gridgen_den(H, W, dev, width=False):
    """The normalisers (s_x, s_y) = ((W - 1) / 2, (H - 1) / 2) as (1, 2, 1, 1); width=True: the control's W / 2, H / 2."""
    k = 0 if width else 1
    return torch.tensor([(W - k) / 2, (H - k) / 2], dtype=torch.float64, device=dev).view(1, 2, 1, 1)


def grid_generator_ref(flow_xy, width=False):
    """(grid, S) of gridgen_warp_kernel in float64: (f + p) / s - 1 and (|f| + p) / s + 1; flow (N, 2, H, W), (x, y)."""
    N, _, H, W = flow_xy.shape
    ys, xs = _pixels(N, H, W, flow_xy.device)
    f, p = flow_xy.double(), torch.stack([xs, ys], 1)
    den = _gridgen_den(H, W, flow_xy.device, width)
    return (f + p) / den - 1, (f.abs() + p) / den + 1


def sampler_positions(grid, H, W):
    """(h, v, dh, dv): the real positions (float64, (N, OH, OW)) the sampler de-normalises the fp32 grid it read to,
    exactly, and how far its fp32 positions fl(fl(g + 1) * (W - 1)) / 2 can lie from them: gamma_2 |v|, gamma_2 |h|."""
    g = grid.double()
    v, h = (g[:, 0] + 1) * ((W - 1) / 2), (g[:, 1] + 1) * ((H - 1) / 2)
    return h, v, gamma(2) * h.abs(), gamma(2) * v.abs()


def _gather_clamped(img, yi, xi):
    """img[n, c, yi, xi] with the indices clamped into the plane: the replicated border."""
    N, C, H, W = img.shape
    idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).reshape(N, 1, -1).expand(N, C, -1)
    return torch.gather(img.reshape(N, C, -1), 2, idx).view(N, C, *yi.shape[1:])


def sampler_forward_bound(img, h, v, dh, dv, replicate=False):
    """(ref, bound) of bilinear_sampler_kernel at the real positions (h, v) with position uncertainty (dh, dv).
    replicate=True: the control that reads an out-of-frame corner as the replicated border (its ref only)."""
    img = img.double()
    y0, x0 = torch.floor(h).long(), torch.floor(v).long()
    gat = _gather_clamped if replicate else _gather0
    a, b, c, d = gat(img, y0, x0), gat(img, y0, x0 + 1), gat(img, y0 + 1, x0), gat(img, y0 + 1, x0 + 1)
    ly, lx = (h - y0).unsqueeze(1), (v - x0).unsqueeze(1)
    ref = (1 - ly) * ((1 - lx) * a + lx * b) + ly * ((1 - lx) * c + lx * d)
    S = (1 - ly) * ((1 - lx) * a.abs() + lx * b.abs()) + ly * ((1 - lx) * c.abs() + lx * d.abs())
    slope_y = slope_x = delta = csum = torch.zeros_like(ref)
    for yy in (torch.floor(h - dh).long(), torch.floor(h + dh).long()):
        for xx in (torch.floor(v - dv).long(), torch.floor(v + dv).long()):
            sy, sx, _, _, dl, cs = sampler_cell_slopes(img, h, v, yy, xx)
            slope_y, slope_x = torch.maximum(slope_y, sy.abs()), torch.maximum(slope_x, sx.abs())
            delta, csum = torch.maximum(delta, dl), torch.maximum(csum, cs)
    dh, dv = dh.unsqueeze(1), dv.unsqueeze(1)
    pos = dh * slope_y + dv * slope_x + delta * dh * dv + 4 * U * csum
    return ref, gamma(SAMPLER_L) * S + pos


def frame_sides(h, v, H, W):
    """The frame sides some sample's corner leaves with a nonzero weight."""
    sides = {"left": (v > -1) & (v < 0), "right": (v > W - 1) & (v < W), "top": (h > -1) & (h < 0),
             "bottom": (h > H - 1) & (h < H)}
    return {k for k, m in sides.items() if bool(m.any())}


def consistency_at_p(flow, other, alpha, beta):
    """The control of mfn_flow_consistency: the other flow read at the pixel p itself instead of at the target q."""
    N, H, W, _ = flow.shape
    y, x = np.mgrid[0:H, 0:W]
    with np.errstate(invalid="ignore", over="ignore"):
        qx = (x.astype(np.float32) + flow[..., 0]).astype(np.float64)
        qy = (y.astype(np.float32) + flow[..., 1]).astype(np.float64)
        inside = (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
        f, g = flow.astype(np.float64), other.astype(np.float64)
        d2 = ((f + g) ** 2).sum(-1)
        rhs = alpha * ((f * f).sum(-1) + (g * g).sum(-1)) + beta
        return ~inside | ~(d2 <= rhs) | ~np.isfinite(rhs)


def _np(t):
    return t.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------------------------------
# GPU: the recorder of the loss-side launches
# ------------------------------------------------------------------------------------------------------------------
class UnsupRecorder:
    """Wraps the launches of losses.unsupervised_loss; rows, controls and failures go to the BackwardRecorder's lists,
    so that its report prints them with the rest."""

    def __init__(self, monkeypatch, bwd):
        self.bwd, self.sides, self.occluded = bwd, set(), []
        for cls, name, fn in ((ops._GridGeneratorWarpFn, "forward", self.gridgen_forward),
                              (ops._GridGeneratorWarpFn, "backward", self.gridgen_backward),
                              (ops._BilinearSamplerFn, "forward", self.sampler_forward),
                              (ops._BilinearSamplerFn, "backward", self.sampler_backward),
                              (ops.CensusLossFn, "forward", self.census_forward),
                              (ops.CensusLossFn, "backward", self.census_backward),
                              (ops.SmoothnessLossFn, "forward", self.smoothness_forward),
                              (ops.SmoothnessLossFn, "backward", self.smoothness_backward)):
            orig = getattr(cls, name)

            def wrapper(ctx, *args, _fn=fn, _orig=orig):
                return _fn(_orig, ctx, *args)
            monkeypatch.setattr(cls, name, staticmethod(wrapper))
        self.orig_consistency = ops.flow_consistency
        monkeypatch.setattr(ops, "flow_consistency", self.consistency)

    def _control_once(self, kind, where, ratios):
        if kind not in self.bwd.controls:
            self.bwd._control(kind, where, ratios)

    # ---- grid generator: gridgen_warp_kernel, gridgen_warp_bwd_kernel ---------------------------------------------
    def gridgen_forward(self, orig, ctx, f):
        grid = orig(ctx, f)
        torch.cuda.synchronize()
        N, _, H, W = f.shape
        with torch.no_grad():
            ref, S = grid_generator_ref(f)
            r, rus, _ = judge_bound(grid, ref, S, GRIDGEN_L)
            self._control_once("gridgen fwd", f"{N}x{H}x{W}",
                               {"W not W-1": judge_bound(grid_generator_ref(f, width=True)[0], ref, S, GRIDGEN_L)[0]})
        self.bwd._row("gridgen_fwd", "grid", f"{N}x2x{H}x{W}", r, rus)
        return grid

    def gridgen_backward(self, orig, ctx, gg):
        gf = orig(ctx, gg)
        torch.cuda.synchronize()
        N, _, H, W = gg.shape
        with torch.no_grad():
            ref = gg.double() / _gridgen_den(H, W, gg.device)
            r, rus, _ = judge_bound(gf, ref, ref.abs(), GRIDGEN_BWD_L)
            ctl = gg.double() / _gridgen_den(H, W, gg.device, width=True)
            self._control_once("gridgen bwd", f"{N}x{H}x{W}", {"W not W-1": judge_bound(ctl, ref, ref.abs(), 1)[0]})
        self.bwd._row("gridgen_bwd", "g_flow", f"{N}x2x{H}x{W}", r, rus)
        return gf

    # ---- bilinear sampler: bilinear_sampler_kernel, bilinear_sampler_bwd_kernel -----------------------------------
    def sampler_forward(self, orig, ctx, d, g):
        out = orig(ctx, d, g)
        torch.cuda.synchronize()
        N, C, H, W = d.shape
        worst, worst_us, ctl = 0.0, 0.0, 0.0
        with torch.no_grad():
            for n in range(N):
                h, v, dh, dv = sampler_positions(g[n:n + 1], H, W)
                self.sides |= frame_sides(h, v, H, W)
                ref, bound = sampler_forward_bound(d[n:n + 1], h, v, dh, dv)
                rmap = _ratio((out[n:n + 1].double() - ref).abs(), bound)
                r = float(rmap.max())
                if r > 1.0:
                    i = int(torch.argmax(rmap))
                    self.bwd.failures.append(f"{self.bwd.run}: sampler fwd n={n} elem {i}: got "
                                             f"{float(out[n:n + 1].reshape(-1)[i]):.9g} ref {float(ref.reshape(-1)[i]):.9g}"
                                             f" bound {float(bound.reshape(-1)[i]):.3g}")
                worst = max(worst, r)
                S = sampler_forward_bound(d[n:n + 1].abs(), h, v, dh * 0, dv * 0)[0]
                worst_us = max(worst_us, float(judge_bound(out[n:n + 1], ref, S, 1)[1]))
                rep = sampler_forward_bound(d[n:n + 1], h, v, dh, dv, replicate=True)[0]
                ctl = max(ctl, float(_ratio((rep - ref).abs(), bound).max()))
        self._control_once("sampler fwd", f"{N}x{C}x{H}x{W}", {"replicated border": ctl})
        self.bwd._row("sampler_fwd", "out", f"{N}x{C}x{H}x{W}", worst, worst_us)
        return out

    def sampler_backward(self, orig, ctx, go):
        res = orig(ctx, go)
        torch.cuda.synchronize()
        gd, gg = res
        d, g = ctx.saved_tensors
        N, C, H, W = d.shape
        if gd is not None:
            self.bwd.failures.append(f"{self.bwd.run}: sampler bwd computed a data gradient the step does not request")
        worst, ctl = 0.0, 0.0
        with torch.no_grad():
            for n in range(N):
                h, v, dh, dv = sampler_positions(g[n:n + 1], H, W)
                r, c, where = image_warp_flow_slopes(d[n:n + 1], h, v, dh, dv, go[n:n + 1], ((H - 1) / 2, (W - 1) / 2),
                                                     gg[n:n + 1].flip(1))
                if r > 1.0:
                    self.bwd.failures.append(f"{self.bwd.run}: sampler bwd n={n}: {where}")
                worst, ctl = max(worst, r), max(ctl, c)
        self._control_once("sampler bwd", f"{N}x{C}x{H}x{W}", {"cell above right": ctl})
        self.bwd._row("sampler_bwd", "g_grid", f"{N}x2x{H}x{W}", worst, 0.0)
        return res

    # ---- census and smoothness: unsup_loss.cu ---------------------------------------------------------------------
    def _unsup_row(self, op, name, shape, got, ref, E):
        r = unsup_ratio(_np(got), ref, E)
        self.bwd._row(op, name, shape, r, r / (1 - 64 * U))
        return r

    def census_forward(self, orig, ctx, img1, img2w, occ):
        loss = orig(ctx, img1, img2w, occ)
        torch.cuda.synchronize()
        ctx.test_occ = occ
        _, _, coef, vsum = ctx.to_save          # save_for_backward's tensors: saved_tensors opens after the forward
        N, _, H, W = img1.shape
        shape = f"{N}x3x{H}x{W}"
        i1, i2, oc = _np(img1), _np(img2w), _np(occ)
        ref = census_bounds(i1, i2, oc, np.ones(N, np.float32))
        if not np.array_equal(_np(vsum), ref["vsum"].numpy().astype(np.float32)):
            self.bwd.failures.append(f"{self.bwd.run}: census vsum differs from the visible-pixel count")
        self._unsup_row("census_fwd", "coef", shape, coef, ref["coef"], ref["E_coef"])
        self._unsup_row("census_fwd", "loss", shape, loss, ref["loss"], ref["E_loss"])
        a, b = torch.from_numpy(i1).double(), torch.from_numpy(i2).double()
        drop = unsup_ref.census_loss(a, b, torch.from_numpy(oc), offsets=unsup_ref.OFFSETS[:-1])[3]
        self._control_once("census fwd", shape, {"dropped offset": unsup_ratio(_np(coef), drop, ref["E_coef"])})
        return loss

    def census_backward(self, orig, ctx, g):
        res = orig(ctx, g)
        torch.cuda.synchronize()
        gi = res[1]
        img1, img2w, _, _ = ctx.saved_tensors
        N, _, H, W = img1.shape
        i1, i2, oc, gl = _np(img1), _np(img2w), _np(ctx.test_occ), _np(g.float())
        with torch.enable_grad():           # the reference's gradient is autograd's; backward runs with it off
            ref = census_bounds(i1, i2, oc, gl)
        self._unsup_row("census_bwd", "g_img2w", f"{N}x3x{H}x{W}", gi, ref["grad"], ref["E_grad"])
        self._control_once("census bwd", f"{N}x3x{H}x{W}", {
            "centre sign flipped": unsup_ratio(_np(gi), census_backward_control(i1, i2, oc, gl), ref["E_grad"])})
        return res

    @staticmethod
    def _other_image(img):
        """[a; b] -> [b; a]: each direction's flow weighted by the other direction's image."""
        n = img.shape[0] // 2
        return torch.cat([img[n:], img[:n]])

    def smoothness_forward(self, orig, ctx, flow, img):
        loss = orig(ctx, flow, img)
        torch.cuda.synchronize()
        N, _, H, W = flow.shape
        ones = np.ones(N, np.float32)
        ref = smoothness_bounds(_np(flow), _np(img), ones)
        self._unsup_row("smoothness_fwd", "loss", f"{N}x2x{H}x{W}", loss, ref["loss"], ref["E_loss"])
        wrong = smoothness_bounds(_np(flow), _np(self._other_image(img)), ones)
        self._control_once("smoothness fwd", f"{N}x2x{H}x{W}",
                           {"other image": unsup_ratio(_np(loss), wrong["loss"], ref["E_loss"])})
        return loss

    def smoothness_backward(self, orig, ctx, g):
        res = orig(ctx, g)
        torch.cuda.synchronize()
        gf = res[0]
        flow, img = ctx.saved_tensors
        N, _, H, W = flow.shape
        gl = _np(g.float())
        with torch.enable_grad():
            ref = smoothness_bounds(_np(flow), _np(img), gl, kernel_signs=True)
            wrong = smoothness_bounds(_np(flow), _np(self._other_image(img)), gl, kernel_signs=True)
        self._unsup_row("smoothness_bwd", "g_flow", f"{N}x2x{H}x{W}", gf, ref["grad"], ref["E_grad"])
        self._control_once("smoothness bwd", f"{N}x2x{H}x{W}",
                           {"other image": unsup_ratio(_np(gf), wrong["grad"], ref["E_grad"])})
        return res

    # ---- forward-backward check: consistency.cu -------------------------------------------------------------------
    def consistency(self, flow_fw, flow_bw, alpha=losses.OCC_ALPHA, beta=losses.OCC_BETA):
        occ = self.orig_consistency(flow_fw, flow_bw, alpha, beta)
        torch.cuda.synchronize()
        fw, bw = _np(flow_fw), _np(flow_bw)
        N, H, W, _ = fw.shape
        ref_fw, ref_bw, amb_fw, amb_bw = consistency_ref(fw, bw, alpha, beta)
        ctl_fw, ctl_bw = consistency_at_p(fw, bw, alpha, beta), consistency_at_p(bw, fw, alpha, beta)
        bad = ctl_bad = excluded = 0
        for got, want, ctl, amb in ((occ[0], ref_fw, ctl_fw, amb_fw), (occ[1], ref_bw, ctl_bw, amb_bw)):
            got = _np(got).astype(bool)
            bad += int(((got != want) & ~amb).sum())
            ctl_bad += int(((got != ctl) & ~amb).sum())
            excluded += int(amb.sum())
            self.occluded.append(float(got.mean()))
        if bad:
            self.bwd.failures.append(f"{self.bwd.run}: flow_consistency: {bad} unambiguous pixels differ from the rule")
        # a wrong decision could hide only among the excluded pixels: the control must disagree on 3x as many
        self._control_once("consistency", f"{N}x{H}x{W}", {"other flow at p": ctl_bad / max(excluded, 1)})
        self.bwd._row("consistency", "mismatches", f"{N}x{H}x{W}", float(bad), excluded / (2 * N * H * W))
        return occ


RUNS = {   # run: (model class, pairs, H, W, image seed) -- tools/finetune_unsupervised.py's defaults first
    "S-4x384x512": (network.MaskFlownetS, 4, 384, 512, 41),
    "S-2x320x768": (network.MaskFlownetS, 2, 320, 768, 46),     # a seed whose flows leave the top row too
    "cascade-1x384x512": (network.MaskFlownet, 1, 384, 512, 43),
}
NEW_KINDS = {   # op: launches per step
    "gridgen_fwd": 2, "gridgen_bwd": 2, "sampler_fwd": 2, "sampler_bwd": 2, "census_bwd": 1, "smoothness_fwd": 1,
    "smoothness_bwd": 1, "consistency": 1}
NEW_CALLS = {
    "mfn_grid_generator_warp_forward": 2, "mfn_grid_generator_warp_backward": 2, "mfn_bilinear_sampler_forward": 2,
    "mfn_bilinear_sampler_backward": 2, "mfn_census_loss_forward": 1, "mfn_census_loss_backward": 1,
    "mfn_smoothness_loss_forward": 1, "mfn_smoothness_loss_backward": 1, "mfn_flow_consistency": 1}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
@pytest.mark.usefixtures("fp64_references")
def test_every_launch_of_the_unsupervised_step_against_float64(run, monkeypatch):
    cls, n, H, W, seed = RUNS[run]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fwd = Recorder(monkeypatch, run)
    bwd = BackwardRecorder(monkeypatch, run)
    rec = UnsupRecorder(monkeypatch, bwd)
    model = _named_model(cls).train()
    with torch.no_grad():
        for k, p in model.named_parameters():
            if "pred_flow" in k or "dc_conv7" in k:
                p.mul_(FLOW_HEAD_SCALE)
    u1, u2 = _images_u8(seed=seed, n=n, h=H, w=W)
    a, b = u1.float() / 255.0, u2.float() / 255.0          # as _train_batch_unsupervised does, without colour augmentation
    x1, x2, _ = network.centralize(torch.cat([a, b]), torch.cat([b, a]))
    preds = model(x1, x2)[0]
    flow = ops.upsample(preds[-1], UPSAMPLE)
    out = losses.unsupervised_loss(a, b, flow[:n], flow[n:], pipeline.SMOOTH_WEIGHT)
    out.loss.sum().backward()
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    monkeypatch.undo()
    fwd.report()
    bwd.report()
    occluded = float(out.occluded.mean())
    print(f"{run}: {len(fwd.rows)} forward and {len(bwd.rows)} backward / loss checks in {secs:.1f} s; occluded "
          f"{occluded:.3f}; max |flow| {float(flow.abs().max()):.3f} px; corners leave the frame on {sorted(rec.sides)}")
    assert not fwd.failures, "\n".join(fwd.failures)
    assert not bwd.failures, "\n".join(bwd.failures)

    # coverage: the graph's launch counts, the frame's four sides, occluded and visible pixels
    for name, k in NEW_CALLS.items():
        assert bwd.calls.count(name) == k, (name, bwd.calls.count(name))
    for op, k in NEW_KINDS.items():
        assert sum(r["op"] == op for r in bwd.rows) == k, op
    assert sum(r["op"] == "census_fwd" for r in bwd.rows) == 2           # coef and loss of its one launch
    cascade = cls is network.MaskFlownet
    assert sum(r["op"] == "corr_bwd" for r in bwd.rows) == 5 + (10 if cascade else 0)
    assert bwd.calls.count("mfn_warp_mask_backward") == 4 + (5 if cascade else 0)
    assert sum(r["op"] == "upsample_bwd" for r in bwd.rows) == 9 + (7 if cascade else 0)
    assert sum(r["op"] == "conv_bwd" for r in bwd.rows) == sum(r["op"] == "conv3x3_slices" for r in fwd.rows)
    assert bwd.calls.count("mfn_image_warp_concat_backward") == (1 if cascade else 0)
    assert rec.sides == {"left", "right", "top", "bottom"}, rec.sides
    assert 0.0 < occluded < 1.0 and len(rec.occluded) == 2, (occluded, rec.occluded)

    # sensitivity: every control fails its bound by CONTROL_MARGIN on a real launch
    want = {"gridgen fwd", "gridgen bwd", "sampler fwd", "sampler bwd", "census fwd", "census bwd", "smoothness fwd",
            "smoothness bwd", "consistency"}
    assert want <= set(bwd.controls), sorted(want - set(bwd.controls))
    for kind, lst in bwd.controls.items():
        for entry in lst:
            assert min(entry[-1].values()) >= CONTROL_MARGIN, (kind, entry)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the sampler and grid generator bounds accept the kernels' arithmetic and reject the controls
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def warp_emu(tmp_path_factory):
    return build(tmp_path_factory, "image_warp_bwd_emu")


def _emu_gridgen(f):
    """gridgen_warp_kernel in fp32, one rounding per operation: fl(fl(fl(f + p) / s) - 1)."""
    N, _, H, W = f.shape
    xs, ys = torch.arange(W, dtype=torch.float32).view(1, 1, W), torch.arange(H, dtype=torch.float32).view(1, H, 1)
    return torch.stack([(f[:, 0] + xs) / ((W - 1) / 2) - 1, (f[:, 1] + ys) / ((H - 1) / 2) - 1], 1)


def _emu_sampler_positions(grid, H, W):
    """The fp32 positions of bilinear_sampler_kernel: fl(fl(g + 1) * (W - 1)) / 2."""
    return (grid[:, 1] + 1) * (H - 1) / 2, (grid[:, 0] + 1) * (W - 1) / 2


def _emu_sampler_forward(img, grid):
    """bilinear_sampler_kernel (sampler_corners, sampling.cuh) in fp32, one rounding per operation."""
    N, C, H, W = img.shape
    yr, xr = _emu_sampler_positions(grid, H, W)
    y0, x0 = torch.floor(yr), torch.floor(xr)
    wx0, wy0 = 1 - (xr - x0), 1 - (yr - y0)
    wx1, wy1 = 1 - wx0, 1 - wy0
    y0, x0 = y0.long(), x0.long()
    out = torch.zeros((N, C, H, W))
    for a, b, wy, wx in ((0, 0, wy0, wx0), (0, 1, wy0, wx1), (1, 0, wy1, wx0), (1, 1, wy1, wx1)):
        ok = (y0 + a >= 0) & (y0 + a <= H - 1) & (x0 + b >= 0) & (x0 + b <= W - 1)
        wt = torch.where(ok, wy * wx, torch.zeros_like(wx)).unsqueeze(1)
        out = out + _gather0(img, y0 + a, x0 + b) * wt
    return out


def test_sampler_bounds_accept_kernel_arithmetic_and_reject_controls(warp_emu):
    """The grid generator's and the sampler's bounds accept the kernels' fp32 arithmetic on flows that reach past all
    four sides of the frame and that land on, and one ulp either side of, integer positions; the controls (the grid
    normalised by W instead of W - 1, the out-of-frame corner read as the replicated border, every slope from the cell
    above and to the right) fail them by CONTROL_MARGIN."""
    g = torch.Generator().manual_seed(14)
    N, C, H, W = 2, 3, 12, 19
    img = torch.rand((N, C, H, W), generator=g)
    f = torch.randn((N, 2, H, W), generator=g) * 0.6                   # (x, y), pixels
    out_by = lambda *s: 0.05 + 0.9 * torch.rand(s, generator=g)  # noqa: E731
    f[:, 0, :, 0], f[:, 0, :, -1] = -out_by(N, H), out_by(N, H)        # left and right columns leave the frame
    f[:, 1, 0, :], f[:, 1, -1, :] = -out_by(N, W), out_by(N, W)        # top and bottom rows too
    xs, ys = torch.arange(W, dtype=torch.float32).view(1, 1, W), torch.arange(H, dtype=torch.float32).view(1, H, 1)
    tx, ty = torch.round(xs + f[:, 0]) - xs, torch.round(ys + f[:, 1]) - ys      # flows to the nearest integers
    inf = torch.tensor(float("inf"))
    for k, t in ((0, tx), (1, ty)):
        f[:, k, 3:5] = t[:, 3:5]                                                    # on an integer
        f[:, k, 5:7] = torch.nextafter(t, inf)[:, 5:7]                              # one ulp either side
        f[:, k, 7:9] = torch.nextafter(t, -inf)[:, 7:9]
    grid = _emu_gridgen(f)
    ref, S = grid_generator_ref(f)
    assert judge_bound(grid, ref, S, GRIDGEN_L)[0] <= 1.0
    assert judge_bound(grid_generator_ref(f, width=True)[0], ref, S, GRIDGEN_L)[0] >= CONTROL_MARGIN
    # rows 9 and 10: grid values one ulp either side of an integer position's, where the sampler's own fp32 position
    # can round onto the integer from the other side
    for k, n_k in ((0, W), (1, H)):
        s_k = (n_k - 1) / 2
        g0 = (torch.round((grid[:, k].double() + 1) * s_k) / s_k - 1).float()
        grid[:, k, 9] = torch.nextafter(g0, inf)[:, 9]
        grid[:, k, 10] = torch.nextafter(g0, -inf)[:, 10]

    h, v, dh, dv = sampler_positions(grid, H, W)
    assert frame_sides(h, v, H, W) == {"left", "right", "top", "bottom"}
    yr, xr = _emu_sampler_positions(grid, H, W)
    # the round trip moved some positions across an integer, and each fp32 position lies within its bound
    assert bool((torch.floor(xr).double() != torch.floor(v)).any() and (torch.floor(yr).double() != torch.floor(h)).any())
    assert bool(((xr.double() - v).abs() <= dv).all() and ((yr.double() - h).abs() <= dh).all())
    out = _emu_sampler_forward(img, grid)
    ref, bound = sampler_forward_bound(img, h, v, dh, dv)
    assert float(_ratio((out.double() - ref).abs(), bound).max()) <= 1.0
    rep = sampler_forward_bound(img, h, v, dh, dv, replicate=True)[0]
    assert float(_ratio((rep - ref).abs(), bound).max()) >= CONTROL_MARGIN

    # the position backward and the grid generator's backward: the kernel source on the host
    go = torch.randn((N, C, H, W), generator=g).numpy()
    gg = np.full((N, 2, H, W), np.nan, np.float32)
    grid_np, img_np = np.ascontiguousarray(grid.numpy()), np.ascontiguousarray(img.numpy())
    warp_emu.emu_bilinear_sampler_backward(ptr(go), ptr(img_np), ptr(grid_np), None, ptr(gg), N, C, H, W, H, W)
    r, ctl, where = image_warp_flow_slopes(img, h, v, dh, dv, torch.from_numpy(go), ((H - 1) / 2, (W - 1) / 2),
                                           torch.from_numpy(gg).flip(1))
    assert r <= 1.0, where
    assert ctl >= CONTROL_MARGIN, ctl
    gf = np.full_like(gg, np.nan)
    warp_emu.emu_grid_generator_warp_backward(ptr(gg), ptr(gf), N, H, W)
    gg64 = torch.from_numpy(gg).double()
    ref = gg64 / _gridgen_den(H, W, "cpu")
    assert judge_bound(torch.from_numpy(gf), ref, ref.abs(), GRIDGEN_BWD_L)[0] <= 1.0
    assert judge_bound(gg64 / _gridgen_den(H, W, "cpu", width=True), ref, ref.abs(), 1)[0] >= CONTROL_MARGIN
