"""Every forward launch against float64 at the shapes a user's own frames reach, and the graph-replayed predictors
against the eager forward.

test_bench_shapes.py checks every launch at the four shapes bench.py times.  network.predict, VideoFlowPredictor and
tools/predict_new_data.py run other shapes -- one pair at a time, KITTI frames (375x1242, padded to 384x1280), HD video
(1080x1920, padded to 1088x1920), images down to 64x64 -- and there the dispatch differs:
  * plan_split (csrc/conv3x3_wgmma.cu) splits every tile at levels 3 and 4 of a single 448x1024 pair, and at level 2 of
    384x1280 and 1088x1920 only the tail rows of the one sample (n_lo = 0);
  * below 4 px ops.warp_mask leaves the through-linearity path: the 2x2 level 5 of a 64x64 pair runs warp_mma_kernel,
    the cascade's 1x1 level-6 warp (F = 196) the SIMT deform_fwd_kernel;
  * the 1x1 correlation has every displacement but the centre outside the image, and the dilation-16 context layer on
    a 16x16 level 2 has every off-centre tap outside: its TMA boxes lie wholly out of bounds.
test_split_plans_of_the_serving_shapes pins those plans on the CPU (mfn_conv3x3_workspace_bytes is host arithmetic).
test_every_launch_of_a_serving_forward_against_float64 runs five forwards through the recorder of test_bench_shapes.py,
with its bound and controls, and asserts that each run reached the path it is there for.  Controls added here, each to
be rejected by CONTROL_MARGIN: replicate padding instead of zero padding (the dilation-16 layer, the 1x1 correlation:
an out-of-bounds box that read the image), the last 16-channel chunk dropped on a split-every-tile launch (a lost
split-K part drops at least that), bf16-only operands and a dropped tap on the warp_mma_kernel launch.  The kitti and hd
runs also compare ops.preprocess (with its resize) and ops.postprocess with oracle/prepost_ref on the same inputs.

The graph paths that give bench.py its numbers, FlowPredictor (a CUDA-graph replay) and PipelinedFlowPredictor (pinned
host buffers, copy streams, staging slots), are compared with the eager forward bit for bit at the benchmark's shapes,
under torch.use_deterministic_algorithms(True): that selects the deterministic preprocessing mean (otherwise the
forward's one run-to-run difference) and fills every torch.empty with NaN, so a kernel that reads a buffer before
writing it shows up as a non-finite or different flow.

Not checked here: the backward at these shapes, frames larger than 1088x1920.
"""
import contextlib
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import _lib, network, ops
from oracle import torch_ref
from test_bench_shapes import (CONTROL_MARGIN, EPS_Q, EPS_S, Recorder, _expected_convs, _images_u8, _named_model,
                               _warp_conv, activate, channel_slopes, conv_terms, judge, split_storage_term)
from make_golden import named_init  # noqa: E402  (tests/golden, on the path test_bench_shapes sets)


# ------------------------------------------------------------------------------------------------------------------
# CPU: the split-K plans the serving runs are there to reach
# ------------------------------------------------------------------------------------------------------------------
def test_split_plans_of_the_serving_shapes():
    """plan_split (csrc/conv3x3_wgmma.cu) for named layers of the serving runs, N = 1: 132 SMs, tiles of 2 rows x 128 px.
    Every tile split when 2 x tiles <= 132: k = min(132 // tiles, chunks // 3, 8) parts, ws = 4 k N Cout OH OW bytes.
    Tail split (a short last round, Cout > 64, >= 16 chunks): the tiles past the last full round of 132, widened to whole
    tile rows, in min(132 // tail, chunks // 2) parts; ws = 4 k Cout rh OW bytes over the rows [OH - rh, OH)."""
    wb = _lib.lib().mfn_conv3x3_workspace_bytes
    # tiny (64x64): every decoder level splits every tile, the 1x1 level 6 included
    assert wb(1, 81, 1, 1, 128, 1, 1) == 2 * 128 * 4                  # conv6_0: 6 chunks -> 2 parts
    assert wb(1, 497, 1, 1, 36, 1, 1) == 8 * 36 * 4                   # conv6_4 + heads
    assert wb(1, 483, 2, 2, 96, 1, 1) == 8 * 96 * 2 * 2 * 4           # conv5_2
    assert wb(1, 451, 4, 4, 96, 1, 1) == 8 * 96 * 4 * 4 * 4           # conv4_2
    assert wb(1, 419, 8, 8, 96, 1, 1) == 8 * 96 * 8 * 8 * 4           # conv3_2
    assert wb(1, 387, 16, 16, 96, 1, 1) == 8 * 96 * 16 * 16 * 4       # conv2_2: 8 tiles
    assert wb(1, 96, 16, 16, 64, 1, 16) == 2 * 64 * 16 * 16 * 4       # dc_conv5, dilation 16: 6 chunks -> 2 parts
    assert wb(1, 32, 16, 16, 2, 1, 1) == 0                             # dc_conv7: 2 chunks, nothing to split
    # single (448x1024): levels 3 (28 tiles) and 4 (14 tiles) split every tile, which batch 8 never does
    assert wb(1, 419, 56, 128, 96, 1, 1) == 4 * 96 * 56 * 128 * 4      # conv3_2: 132 // 28 = 4
    assert wb(1, 451, 28, 64, 96, 1, 1) == 8 * 96 * 28 * 64 * 4        # conv4_2: min(132 // 14, 29 // 3, 8)
    assert wb(1, 195, 28, 64, 128, 1, 1) == 4 * 128 * 28 * 64 * 4      # conv4_0: 13 chunks -> 4
    assert wb(1, 579, 112, 256, 128, 1, 1) == 0                        # level 2: 112 tiles, one short round
    # kitti (384x1280): level 2 is 96x320, 3 tiles per row (2.5 tiles of pixels), 144 tiles = 132 + 12: the last 12 are
    # tile rows 44..47 = rows 88..95 of the only sample, in 132 // 12 = 11 parts
    assert wb(1, 387, 96, 320, 96, 1, 1) == 11 * 96 * 8 * 320 * 4      # conv2_2
    assert wb(1, 579, 96, 320, 128, 1, 1) == 11 * 128 * 8 * 320 * 4    # dc_conv1
    assert wb(1, 259, 96, 320, 128, 1, 1) == 8 * 128 * 8 * 320 * 4     # conv2_1: 17 chunks -> 8
    assert wb(1, 483, 96, 320, 64, 1, 1) == 0                          # conv2_3: Cout 64 does not gain
    # hd (1088x1920): level 2 is 272x480, 4 tiles per row (3.75), 544 tiles = 4 x 132 + 16: tile rows 132..135 = rows
    # 264..271 in 132 // 16 = 8 parts; level 3 (136x240, 136 tiles = 132 + 4): rows 132..135 in 19 // 2 = 9 parts
    assert wb(1, 579, 272, 480, 128, 1, 1) == 8 * 128 * 8 * 480 * 4    # dc_conv1
    assert wb(1, 387, 272, 480, 96, 1, 1) == 8 * 96 * 8 * 480 * 4      # conv2_2
    assert wb(1, 291, 136, 240, 128, 1, 1) == 9 * 128 * 4 * 240 * 4    # conv3_1
    # level 6 is 17x30 (odd height, rows of 30 px): 9 tiles, every tile split
    assert wb(1, 337, 17, 30, 96, 1, 1) == 7 * 96 * 17 * 30 * 4        # conv6_2: 21 chunks -> 7


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound holds for a bias-dominated output stored as a split activation
# ------------------------------------------------------------------------------------------------------------------
def test_split_output_storage_term_covers_a_bias_dominated_output():
    """conv6_0 on a 1x1 level 6: the md=4 correlation input is zero but for the centre displacement, so Q = |w x| is
    tiny and the output is nearly the bias.  The kernel's arithmetic (hi/lo split operands, fp32 sums, LeakyReLU) with
    an fp32 output passes 2^-12 Q + 2^-20 S; stored as a split activation (bf16 hi + lo of the fp32 value) it needs the
    storage term 2^-16 |ref| of split_storage_term, which it then passes."""
    w = named_init("conv6_0.weight", (128, 81, 3, 3))
    b = named_init("conv6_0.bias", (128,))
    sl = channel_slopes(128, 0.1)

    def split(t):
        hi = t.bfloat16().float()
        return hi, (t - hi).bfloat16().float()
    worst = {"fp32": 0.0, "split, no term": 0.0, "split": 0.0}
    for v in (0.0123, -0.0071, 0.031, 0.0042):
        x = torch.zeros((1, 81, 1, 1))
        x[0, 40] = v
        (xh, xl), (wh, wl) = split(x), split(w)
        conv32 = lambda p, q: tF.conv2d(p, q, padding=1)  # noqa: E731
        out = tF.leaky_relu(conv32(xh, wh) + conv32(xh, wl) + conv32(xl, wh) + b.view(1, -1, 1, 1), 0.1)
        oh, ol = split(out)
        pre, Q, S = conv_terms(x.double(), w.double(), b.double())
        bound = EPS_Q * Q + EPS_S * S
        worst["fp32"] = max(worst["fp32"], judge(out, pre, sl, bound, Q)[0])
        worst["split, no term"] = max(worst["split, no term"], judge(oh.double() + ol.double(), pre, sl, bound, Q)[0])
        worst["split"] = max(worst["split"], judge(oh.double() + ol.double(), pre, sl,
                                                   bound + split_storage_term(pre, 0), Q)[0])
    assert worst["fp32"] <= 1.0 and worst["split"] <= 1.0 and worst["split, no term"] > 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: the recorder with this file's controls
# ------------------------------------------------------------------------------------------------------------------
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
    """test_bench_shapes.Recorder plus: where each launch's split-K plan splits every tile, the controls of this file
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


# ------------------------------------------------------------------------------------------------------------------
# GPU: the five serving forwards
# ------------------------------------------------------------------------------------------------------------------
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


def _cover_single(rec, convs):
    for h in (56, 28):      # levels 3 and 4
        split = [r for r in convs if r["op"] == "conv3x3_split" and r["H"] == h and r["ws"] > 0]
        assert len(split) >= 5 and all(r["split_all"] and r["N"] == 1 for r in split), (h, split)
    assert "chunk" in rec.extra


def _tail_rows_8(r):
    """A tail split of rows [OH - 8, OH) of the only sample: ws = 4 k Cout 8 OW."""
    return r["ws"] > 0 and not r["split_all"] and r["ws"] % (4 * r["Cout"] * 8 * r["W"]) == 0


def _cover_prepost(rec, net_hw):
    pre = [r for r in rec.rows if r["op"] == "preprocess"]
    post = [r for r in rec.rows if r["op"] == "postprocess"]
    assert len(pre) == 1 and pre[0]["name"] == f"-> {net_hw[0]}x{net_hw[1]}" and len(post) == 2


def _cover_kitti(rec, convs):
    lvl2 = [r for r in convs if r["op"] == "conv3x3_split" and (r["H"], r["W"]) == (96, 320)]
    assert lvl2 and sum(_tail_rows_8(r) for r in lvl2) >= 3, lvl2    # conv2_1, conv2_2, dc_conv1: rows 88..95
    _cover_prepost(rec, (384, 1280))


def _cover_hd(rec, convs):
    # an odd-height level 6 with 30-px rows, fp32 outputs included (rows of 30 floats are not 16-byte aligned, which by
    # conv3x3_wgmma_launch's `staged` condition sends them to the register epilogue; which epilogue ran is not
    # observable from here, only that these launches ran and were checked)
    assert any((r["H"], r["W"]) == (17, 30) and not r["split_out"] for r in convs)
    lvl2 = [r for r in convs if r["op"] == "conv3x3_split" and (r["H"], r["W"]) == (272, 480)]
    assert lvl2 and sum(_tail_rows_8(r) for r in lvl2) >= 3, lvl2    # rows 264..271
    _cover_prepost(rec, (1088, 1920))


SERVING = {   # run: (model class, batch, input H, W, image seed, through network.predict, coverage)
    "tiny": (network.MaskFlownetS, 1, 64, 64, 31, False, _cover_tiny),
    "tiny_cascade": (network.MaskFlownet, 1, 64, 64, 32, False, _cover_tiny_cascade),
    "single": (network.MaskFlownetS, 1, 448, 1024, 33, False, _cover_single),
    "kitti": (network.MaskFlownetS, 1, 375, 1242, 34, True, _cover_kitti),
    "hd": (network.MaskFlownetS, 1, 1080, 1920, 35, True, _cover_hd),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(SERVING))
def test_every_launch_of_a_serving_forward_against_float64(run, monkeypatch):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    cls, N, H, W, seed, via_predict, cover = SERVING[run]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    rec = ServingRecorder(monkeypatch, run)         # before the model packs anything
    model = _named_model(cls).eval()
    u1, u2 = _images_u8(seed=seed, n=N, h=H, w=W)
    if via_predict:
        flow, occ = network.predict(model, u1, u2)
        assert flow.shape == (N, H, W, 2) and occ.shape == (N, H, W, 1)
    else:
        flow = network.predict_flow(model, u1, u2)
        assert flow.shape == (N, 2, H, W)
    assert bool(torch.isfinite(flow).all())
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    rec.report()
    print(f"{run}: {len(rec.rows)} launches checked in {secs:.1f} s, peak {peak:.2f} GiB allocated")
    assert not rec.failures, "\n".join(rec.failures)

    convs = [r for r in rec.rows if r["op"] in ("conv3x3_slices", "conv3x3_split")]
    assert len(convs) == _expected_convs("cascade" if cls is network.MaskFlownet else "fwd"), len(convs)
    assert set(Recorder.KINDS) <= set(rec.controls), sorted(rec.controls)
    for tag, (name, rs) in rec.controls.items():
        assert min(rs.values()) >= CONTROL_MARGIN, (tag, name, rs)
    for tag, (name, r) in rec.extra.items():
        assert r >= CONTROL_MARGIN, (tag, name, r)
    cover(rec, convs)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the serving paths against eager, bit for bit
# ------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _same(got, ref, what):
    assert bool(torch.isfinite(ref).all()), f"{what}: the eager flow is not finite"
    d = (got.float() - ref.float()).abs()
    assert torch.equal(got, ref), f"{what}: max |diff| {float(d.nan_to_num(float('inf')).max()):.3g} at " \
                                  f"{np.unravel_index(int(d.nan_to_num(float('inf')).argmax()), tuple(d.shape))}"


@pytest.mark.gpu
@pytest.mark.parametrize("arch,N,conv,deform", [("S", 8, "conv5_1", "deform4"), ("cascade", 4, "conv4_1", "deform3")])
def test_flow_predictor_graph_equals_eager_at_the_benchmark_shape(arch, N, conv, deform):
    """FlowPredictor (bench.py's judged value) replays the eager forward bit for bit: on two pairs, on the first again
    after the second, and after an in-place weight change followed by invalidate()."""
    model = _named_model(network.MaskFlownetS if arch == "S" else network.MaskFlownet).eval()
    p1 = _images_u8(seed=41, n=N, h=448, w=1024)
    p2 = _images_u8(seed=42, n=N, h=448, w=1024)
    with _deterministic():
        e1 = network.predict_flow(model, *p1).clone()
        _same(network.predict_flow(model, *p1), e1, f"{arch}: eager twice")
        e2 = network.predict_flow(model, *p2).clone()
        pred = network.FlowPredictor(model)
        _same(pred(*p1), e1, f"{arch}: graph, pair 1")
        _same(pred(*p2), e2, f"{arch}: graph, pair 2")
        _same(pred(*p1), e1, f"{arch}: graph, pair 1 after pair 2")
        with torch.no_grad():
            getattr(model, conv).weight.mul_(1.25)
            getattr(model, deform).weight.mul_(0.75)
        pred.invalidate()
        e3 = network.predict_flow(model, *p1).clone()
        assert not torch.equal(e3, e1), "the weight change did not change the flow"
        _same(pred(*p1), e3, f"{arch}: graph after the weight change")
        torch.cuda.synchronize()


@pytest.mark.gpu
def test_pipelined_predictor_equals_eager_at_the_benchmark_shape():
    """PipelinedFlowPredictor(depth=2): five distinct pinned pairs enqueued into five pinned outputs without a
    synchronisation in between; the last output is complete once the event its infer() returned has completed, and every
    output equals the eager flow after synchronize()."""
    model = _named_model(network.MaskFlownetS).eval()
    with _deterministic():
        pairs, refs = [], []
        for i in range(5):
            a, b = _images_u8(seed=50 + i, n=8, h=448, w=1024)
            refs.append(network.predict_flow(model, a, b).cpu())
            pairs.append((a.cpu().pin_memory(), b.cpu().pin_memory()))
        outs = [torch.full((8, 2, 448, 1024), float("nan")).pin_memory() for _ in range(5)]
        pipe = network.PipelinedFlowPredictor(model, depth=2)
        torch.cuda.synchronize()
        evs = [pipe.infer(a, b, o) for (a, b), o in zip(pairs, outs)]
        evs[-1].synchronize()
        _same(outs[-1], refs[-1], "pipelined: last output after its event")
        pipe.synchronize()
        for i in range(5):
            _same(outs[i], refs[i], f"pipelined: request {i}")


@pytest.mark.gpu
def test_pipelined_predictor_gives_each_shape_its_own_slots():
    """A batch-8 request at 448x1024, a batch-2 request at 64x128 (a 1x2 level 6), then batch 8 again: each equals the
    eager flow."""
    model = _named_model(network.MaskFlownetS).eval()
    reqs = [_images_u8(seed=60, n=8, h=448, w=1024), _images_u8(seed=61, n=2, h=64, w=128),
            _images_u8(seed=62, n=8, h=448, w=1024)]
    with _deterministic():
        refs = [network.predict_flow(model, a, b).cpu() for a, b in reqs]
        host = [(a.cpu().pin_memory(), b.cpu().pin_memory()) for a, b in reqs]
        outs = [torch.full(tuple(r.shape), float("nan")).pin_memory() for r in refs]
        pipe = network.PipelinedFlowPredictor(model, depth=2)
        for (a, b), o in zip(host, outs):
            pipe.infer(a, b, o)
        pipe.synchronize()
        for i, (o, r) in enumerate(zip(outs, refs)):
            _same(o, r, f"pipelined: request {i} {tuple(r.shape)}")
