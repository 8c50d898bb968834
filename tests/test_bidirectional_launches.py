"""Every launch of the bidirectional forward (network.predict_bidirectional) against float64, at the video tools' batch
and frame sizes.

Occlusion masks, frame interpolation, point tracking and stabilisation all run `net(a, b, bidirectional=True)`, and the
video tools default to 8 pairs per batch.  That forward runs one pyramid pass over [im1; im2] and every correlation,
warp, decoder and context layer at batch 2N = 16 (the cascade's dual pyramid too).  At 8 pairs of 1080p frames (padded
to 1088x1920) the dispatch differs from every shape test_bench_shapes.py and test_serving_shapes.py check:
  * plan_split (csrc/conv3x3_wgmma.cu) splits the tail of levels 5 and 4 inside the last sample (n_lo = 15, the
    backward half's last pair) and no tile at levels 6, 3 and 2, where one pair splits every tile or a tail;
  * MaskFlownet-S's level-2 dense-block buffer (ops.SplitAct, 579 channels) holds about 309 MB per sample, so from
    sample 14 on its entries lie past 2^32 bytes.
test_split_plans_of_the_bidirectional_shapes pins those plans on the CPU (mfn_conv3x3_workspace_bytes is host
arithmetic).  test_every_launch_of_a_bidirectional_forward_against_float64 runs predict_bidirectional through
ServingRecorder (launchcheck.recorders: the float64 recorder of test_bench_shapes.py, its bounds and controls, and
pre- / post-processing against oracle/prepost_ref), extended here with:
  * ops.flow_consistency against launchcheck.bidirectional.consistency_ref outside the ambiguous pixels;
  * the wiring, bit for bit, which per-launch judging cannot see (each launch is judged on the inputs it read): the
    first pyramid launch reads the ops.preprocess buffer in place; every S-head correlation reads the pyramid output as
    its first operand, and at level 6 its halves swapped as its second; every S-head warp warps the swapped pyramid
    level; the cascade's warps read the swapped level at levels 6..4 and the unswapped one at levels 3 and 2 (the
    reference's c2s quirk, network.MaskFlownetS.forward); the cascade's image_warp_concat reads im2 = im1 with its
    halves swapped;
  * controls, each to fail by CONTROL_MARGIN: a backward-half level-6 correlation judged against the reference built
    from the unswapped second operand; the last 16-channel chunk dropped in the last tile row of the last sample on the
    first tail-split launch (the smallest region a lost split-K part of the tail would touch); and on the first pair,
    the rule's decisions with flow_fw and flow_bw exchanged must differ from the kernel's, outside both ambiguous sets,
    on at least CONTROL_MARGIN times as many pixels as the comparison excludes there.  The rule is symmetric in the two
    flows to first order (|u + u'(x + u)| against |u' + u(x + u')|), so on smooth flows the exchange changes only the
    decisions near the threshold and at the frame's edges: about 0.3 % of them at 1080p for MaskFlownet-S, 0.05 % for
    the cascade, whose flows leave almost every pixel occluded.  A share of the pixels (a multiple of AMBIGUOUS_MAX)
    would ask more of this control than such flows give; the count it is held to is what the comparison could hide.
The flow heads are scaled by launchcheck.inputs.FLOW_HEAD_SCALE, so that the occluded share of each direction lies
strictly inside (0, 1) and both decisions are reached.  hd8 runs once more in bf16 mode under BF16Recorder
(test_bf16_mode.py), and VideoFlowPredictor(bidirectional=True) must replay its eager chain bit for bit at batch 8 on a
9-frame 1080p clip.

Not checked here: frames larger than 1088x1920; the kernels of the video tools that follow this forward (interpolation,
tracking, stabilisation and motion segmentation): test_video_chain_launches.py checks every one of their launches in
the tools' chains against float64 at batch 8 on 1080p, and which pair each frame reads; test_denoise_chain_launches.py
does the same for video denoising (network.denoise_video and VideoDenoiser's ring).
"""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import _lib, network, ops
from maskflownet_b200.video import VideoFlowPredictor
from oracle import torch_ref

from launchcheck import fp64_references  # noqa: F401
from launchcheck.bidirectional import AMBIGUOUS_MAX, consistency_ref
from launchcheck.bounds import (CONTROL_MARGIN, EPS_Q, EPS_S, _expected_convs, activate, channel_slopes, conv_terms,
                                judge, split_storage_term)
from launchcheck.inputs import _clip, _deterministic, _images_u8, _same, _scaled_model
from launchcheck.recorders import BF16Recorder, Recorder, ServingRecorder, _cover_tiny, _cover_tiny_cascade

HD_CASCADE_PAIRS = 8


# ------------------------------------------------------------------------------------------------------------------
# CPU: the split-K plans of the decoder batch 2N
# ------------------------------------------------------------------------------------------------------------------
def test_split_plans_of_the_bidirectional_shapes():
    """plan_split for named layers at the decoder batch 2N (132 SMs, tiles of 2 rows x MT px, MT = 64 where the output
    is at most 64 px wide, else 128).  Every tile split when 2 x tiles <= 132: k = min(132 // tiles, chunks // 3, 8),
    ws = 4 k 2N Cout OH OW bytes.  Tail split (a short last round, at most 12 rounds, Cout > 64, >= 16 chunks, the tail
    widened to whole tile rows and no longer than one sample): k = min(132 // tail, chunks // 2) parts over the rows
    [OH - rh, OH) of the last sample, ws = 4 k Cout rh OW."""
    wb = _lib.lib().mfn_conv3x3_workspace_bytes
    # hd8 (8 pairs of 1088x1920 -> 16 decoders), MaskFlownet-S
    # level 6 (17x30): 1 x 9 tiles per sample, 144 = 132 + 12 tiles; the 12-tile tail spans two samples: no split
    assert wb(16, 209, 17, 30, 128, 1, 1) == 0                           # conv6_1
    assert wb(16, 337, 17, 30, 96, 1, 1) == 0                            # conv6_2
    # level 5 (34x60): 1 x 17 tiles per sample, 272 = 2 x 132 + 8: tile rows 9..16 = rows 18..33 of sample 15,
    # in min(132 // 8, chunks // 2) parts
    assert wb(16, 227, 34, 60, 128, 1, 1) == 0                           # conv5_0: 15 chunks, fewer than 16
    assert wb(16, 355, 34, 60, 128, 1, 1) == 11 * 128 * 16 * 60 * 4      # conv5_1: 23 chunks -> 11
    assert wb(16, 483, 34, 60, 96, 1, 1) == 15 * 96 * 16 * 60 * 4        # conv5_2: 31 chunks -> 15
    assert wb(16, 579, 34, 60, 64, 1, 1) == 0                            # conv5_3: Cout 64 does not gain
    # level 4 (68x120): 1 x 34 tiles per sample, 544 = 4 x 132 + 16: tile rows 18..33 = rows 36..67 of sample 15,
    # in 132 // 16 = 8 parts
    assert wb(16, 323, 68, 120, 128, 1, 1) == 8 * 128 * 32 * 120 * 4     # conv4_1: 21 chunks
    assert wb(16, 451, 68, 120, 96, 1, 1) == 8 * 96 * 32 * 120 * 4       # conv4_2: 29 chunks
    # level 3 (136x240): 2 x 68 tiles, 2176 tiles = 16 rounds + 64, more than 12 rounds; level 2 (272x480): 8704 tiles
    assert wb(16, 419, 136, 240, 96, 1, 1) == 0                          # conv3_2
    assert wb(16, 387, 272, 480, 96, 1, 1) == 0                          # conv2_2
    assert wb(16, 579, 272, 480, 128, 1, 1) == 0                         # dc_conv1
    # the 196-channel pyramid layers (two 128-channel halves per tile) split only small images
    assert wb(16, 196, 17, 30, 196, 1, 1) == 0                           # conv6b
    # hd_cascade at 16: the cascade's own dense blocks split the same tails (level 5: 198 input channels, level 4: 166)
    assert wb(16, 326, 34, 60, 128, 1, 1) == 10 * 128 * 16 * 60 * 4      # conv5_1: 21 chunks -> 10
    assert wb(16, 454, 34, 60, 96, 1, 1) == 14 * 96 * 16 * 60 * 4        # conv5_2: 29 chunks -> 14
    assert wb(16, 294, 68, 120, 128, 1, 1) == 8 * 128 * 32 * 120 * 4     # conv4_1: 19 chunks -> 8
    assert wb(16, 422, 68, 120, 96, 1, 1) == 8 * 96 * 32 * 120 * 4       # conv4_2
    # kitti4 (4 pairs of 384x1280 -> 8 decoders): levels 6 (6x20, 24 tiles) and 5 (12x40, 48 tiles) split every tile;
    # level 2 (96x320, 3 x 48 tiles per sample): 1152 = 8 x 132 + 96, and 132 // 96 = 1 part is no split
    assert wb(8, 337, 6, 20, 96, 1, 1) == 5 * 8 * 96 * 6 * 20 * 4       # conv6_2: 132 // 24 = 5
    assert wb(8, 483, 12, 40, 96, 1, 1) == 2 * 8 * 96 * 12 * 40 * 4     # conv5_2: 132 // 48 = 2
    assert wb(8, 387, 96, 320, 96, 1, 1) == 0                            # conv2_2
    # tiny (1 pair of 64x64 -> 2 decoders): every tile split at every level, the 1x1 level 6 included
    assert wb(2, 81, 1, 1, 128, 1, 1) == 2 * 2 * 128 * 4                 # conv6_0: 6 chunks -> 2 parts
    assert wb(2, 497, 1, 1, 36, 1, 1) == 8 * 2 * 36 * 4                  # conv6_4 + heads: 2 tiles, 32 chunks -> 8
    assert wb(2, 483, 2, 2, 96, 1, 1) == 8 * 2 * 96 * 2 * 2 * 4          # conv5_2: 2 tiles
    assert wb(2, 451, 4, 4, 96, 1, 1) == 8 * 2 * 96 * 4 * 4 * 4          # conv4_2: 4 tiles
    assert wb(2, 419, 8, 8, 96, 1, 1) == 8 * 2 * 96 * 8 * 8 * 4          # conv3_2: 8 tiles
    assert wb(2, 387, 16, 16, 96, 1, 1) == 8 * 2 * 96 * 16 * 16 * 4      # conv2_2: 16 tiles
    assert wb(2, 96, 16, 16, 64, 1, 16) == 2 * 2 * 64 * 16 * 16 * 4      # dc_conv5, dilation 16: 6 chunks -> 2
    assert wb(2, 32, 16, 16, 2, 1, 1) == 0                               # dc_conv7: 2 chunks, nothing to split


# ------------------------------------------------------------------------------------------------------------------
# GPU: the recorder with this file's checks
# ------------------------------------------------------------------------------------------------------------------
def _is_swap(t, p, n):
    """t == [p[n:]; p[:n]] bit for bit."""
    return t.shape == p.shape and torch.equal(t[:n], p[n:]) and torch.equal(t[n:], p[:n])


def _same_tensor(t, p):
    return t.data_ptr() == p.data_ptr() and t.shape == p.shape and t.stride() == p.stride()


class BidirRecorder(ServingRecorder):
    """ServingRecorder plus: ops.flow_consistency against the oracle, the bidirectional wiring bit for bit
    (self.wiring: description -> ok), the split activations' sizes, and this file's controls in self.extra."""

    def __init__(self, monkeypatch, run, n):
        super().__init__(monkeypatch, run)
        self.n = n                  # pairs: the forward runs at batch 2n
        self.pyr = {}               # pyramid level -> output of S.conv{L}c, the 2n-sample [f(im1); f(im2)]
        self.pair = None            # the ops.preprocess buffer's first half
        self.wiring = {}
        self.max_act_bytes = 0
        self.occluded = None
        self.exchanged = None       # (decisions changed, pixels excluded, pixels) on the first pair
        self.orig["flow_consistency"] = ops.flow_consistency
        monkeypatch.setattr(ops, "flow_consistency", self.flow_consistency)

    def _wire(self, what, ok):
        self.wiring[what] = bool(ok)
        if not ok:
            self._fail(f"wiring: {what}")

    def _level_of(self, t):
        return next((L for L, p in self.pyr.items() if p.shape[2:] == t.shape[2:]), None)

    # ---- the pyramid: the preprocess buffer in place, and its outputs ---------------------------------------------
    def preprocess(self, img1, img2, out_hw=None):
        res = super().preprocess(img1, img2, out_hw)
        self.pair = res[0]
        return res

    def conv3x3_slices(self, *args, **kw):
        a = self._bind("conv3x3_slices", args, kw)
        if "first pyramid launch reads the preprocess buffer in place" not in self.wiring:
            x, p = a["buf_in"], self.pair
            self._wire("first pyramid launch reads the preprocess buffer in place",
                       p is not None and x.data_ptr() == p.data_ptr() and x.shape[0] == 2 * self.n and
                       x.shape[1:] == p.shape[1:])
        super().conv3x3_slices(*args, **kw)
        name = self.names.get(a["packed"].data_ptr(), "?")
        if name.startswith("S.conv") and name.endswith("c"):
            self.pyr[int(name[len("S.conv")])] = a["buf_out"]

    def conv3x3_split(self, *args, **kw):
        a = self._bind("conv3x3_split", args, kw)
        self.max_act_bytes = max(self.max_act_bytes, a["x"].buf.numel())
        super().conv3x3_split(*args, **kw)

    # ---- the tail control: the last chunk dropped in the last tile row of the last sample --------------------------
    def _check_conv(self, op, packed, bias, Cout, slope, dil, stride, d2s, lp, x_of, got_of, N, Cin, H, W, ws, kern,
                    tags, store_from=None):
        super()._check_conv(op, packed, bias, Cout, slope, dil, stride, d2s, lp, x_of, got_of, N, Cin, H, W, ws, kern,
                            tags, store_from)
        row = self.rows[-1]
        if ws and not row["split_all"] and not d2s and Cin > 16 and "tail_chunk" not in self.extra:
            w = self.packs[packed.data_ptr()][0].double()
            b = bias.detach().double() if bias is not None else None
            sl = channel_slopes(Cout, slope, lp, w.device)
            with torch.no_grad():
                x = x_of(N - 1)
                pre, Q, S = conv_terms(x, w, b, stride, dil)
                bound = EPS_Q * Q + EPS_S * S + split_storage_term(pre, store_from)
                wd = w.clone()
                wd[:, (Cin - 1) // 16 * 16:] = 0
                alt = pre.clone()
                alt[:, :, -2:] = tF.conv2d(x, wd, stride=stride, padding=dil, dilation=dil)[:, :, -2:] + \
                    (b.view(1, -1, 1, 1) if b is not None else 0.0)
                r = judge(activate(alt, sl), pre, sl, bound, Q)[0]
                self.extra["tail_chunk"] = (f"{row['name']} sample {N - 1}", r)

    # ---- correlation and warp: which operands they read --------------------------------------------------------------
    def correlation(self, *args, **kw):
        res = super().correlation(*args, **kw)
        a = self._bind("correlation", args, kw)
        d1, d2, md = a["data1"], a["data2"], a["max_displacement"]
        L, n = self._level_of(d1), self.n
        if L is None or not _same_tensor(d1, self.pyr[L]):
            if md == 4:
                self._fail(f"correlation md=4 {tuple(d1.shape)}: the first operand is not a pyramid output")
            return res            # the cascade's correlation of its dual pyramid
        who = "S" if md == 4 else "cascade"
        self._wire(f"{who} correlation L{L}: first operand is the pyramid output", True)
        if md == 4 and L == 6:
            P = self.pyr[6]
            self._wire("S correlation L6: second operand is the pyramid output, halves swapped", _is_swap(d2, P, n))
            if "unswapped" not in self.extra:     # the last backward-half sample judged against (f(im1), f(im1))
                k = 2 * n - 1
                with torch.no_grad():
                    f1, f2, fu = (t[k:k + 1].detach().double() for t in (d1, d2, P))
                    C = f1.shape[1]
                    pre = torch_ref.correlation(f1, f2, md)
                    Q = (torch_ref.correlation(f1 * f1, f2 * f2, md) * C).sqrt() / C
                    S = torch_ref.correlation(f1.abs(), f2.abs(), md)
                    sl = channel_slopes(pre.shape[1], a["leaky_slope"], 0, d1.device)
                    alt = activate(torch_ref.correlation(f1, fu, md), sl)
                    r = judge(alt, pre, sl, EPS_Q * Q + EPS_S * S, Q)[0]
                    self.extra["unswapped"] = (f"correlation L6 sample {k}", r)
        return res

    def warp_mask(self, *args, **kw):
        res = super().warp_mask(*args, **kw)
        a = self._bind("warp_mask", args, kw)
        name = self.names.get(a["packed_weight"].data_ptr(), "?") if a["packed_weight"] is not None else "?"
        x, L = a["x"], int(name[-1]) if name[-1].isdigit() else None
        if L not in self.pyr:
            self._fail(f"warp_mask {name}: no pyramid level {L}")
        elif name.startswith("cascade.") and L <= 3:     # c2s carries image-1 features at levels 2 and 3
            self._wire(f"{name}: warps the unswapped pyramid output", _same_tensor(x, self.pyr[L]))
        else:
            self._wire(f"{name}: warps the pyramid output, halves swapped", _is_swap(x, self.pyr[L], self.n))
        return res

    def image_warp_concat(self, *args, **kw):
        a = self._bind("image_warp_concat", args, kw)
        im1, im2 = a["im1"], a["im2"]
        self._wire("image_warp_concat: im1 is the preprocess buffer", self.pair is not None and
                   im1.data_ptr() == self.pair.data_ptr() and im1.shape[0] == 2 * self.n)
        self._wire("image_warp_concat: im2 is im1, halves swapped", _is_swap(im2, im1, self.n))
        return super().image_warp_concat(*args, **kw)

    # ---- the consistency check against the float64 rule -------------------------------------------------------------
    def flow_consistency(self, flow_fw, flow_bw, alpha=0.01, beta=0.5):
        res = self.orig["flow_consistency"](flow_fw, flow_bw, alpha, beta)
        torch.cuda.synchronize()
        kern = _lib.last_kernel()
        fw, bw = flow_fw.cpu().numpy(), flow_bw.cpu().numpy()
        got = [t.cpu().numpy().astype(bool) for t in res]
        occ_fw, occ_bw, amb_fw, amb_bw = consistency_ref(fw, bw, alpha, beta)
        bad = int(((got[0] != occ_fw) & ~amb_fw).sum() + ((got[1] != occ_bw) & ~amb_bw).sum())
        excluded, total = int(amb_fw.sum() + amb_bw.sum()), 2 * occ_fw.size
        if bad or excluded > AMBIGUOUS_MAX * total:
            self._fail(f"flow_consistency {fw.shape}: {bad} pixels differ, {excluded} of {total} excluded")
        # control on the first pair: the decisions of the rule with the two flows exchanged
        x_fw, x_bw, xa_fw, xa_bw = consistency_ref(bw[:1], fw[:1], alpha, beta)
        differ = int(((got[0][:1] != x_fw) & ~xa_fw & ~amb_fw[:1]).sum() +
                     ((got[1][:1] != x_bw) & ~xa_bw & ~amb_bw[:1]).sum())
        self.exchanged = (differ, int(amb_fw[:1].sum() + amb_bw[:1].sum()), 2 * x_fw.size)
        self.occluded = (float(got[0].mean()), float(got[1].mean()))
        N, H, W, _ = fw.shape
        self.rows.append(dict(op="flow_consistency", name=f"{excluded} excluded", kernel=kern, N=N, Cin=2, Cout=1, H=H,
                              W=W, dil=0, stride=1, ws=0, err_q=0.0, ratio=float(bad), tags=[], split_out=False))
        return res

    def report(self):
        super().report()
        for what, ok in self.wiring.items():
            print(f"{self.run:8s} wiring {'ok ' if ok else 'BAD'} {what}")
        if self.occluded is not None:
            d, e, t = self.exchanged
            print(f"{self.run:8s} occluded fw {self.occluded[0]:.3f} bw {self.occluded[1]:.3f}; on the first pair the "
                  f"exchanged flows change {d} of {t} decisions ({d / t:.4f}), {e} excluded")
        print(f"{self.run:8s} largest split activation {self.max_act_bytes / 2 ** 30:.2f} GiB")


# ------------------------------------------------------------------------------------------------------------------
# GPU: the runs
# ------------------------------------------------------------------------------------------------------------------
def _tails(convs, N):
    return {r["name"]: r for r in convs if r["ws"] > 0 and not r["split_all"] and r["N"] == N}


def _tail_rows(r, rh):
    """A tail split of rows [OH - rh, OH) of the last sample alone: ws = 4 k Cout rh OW."""
    return r["ws"] % (4 * r["Cout"] * rh * r["W"]) == 0 and r["ws"] // (4 * r["Cout"] * rh * r["W"]) >= 2


def _cover_hd8(rec, convs):
    tails = _tails(convs, 16)
    assert set(tails) == {"S.conv5_1", "S.conv5_2", "S.conv4_1", "S.conv4_2"}, sorted(tails)
    assert all(_tail_rows(tails[f"S.conv5_{i}"], 16) and _tail_rows(tails[f"S.conv4_{i}"], 32) for i in (1, 2)), tails
    assert not any(r["split_all"] for r in convs)
    assert any((r["H"], r["W"]) == (17, 30) for r in convs)
    assert rec.max_act_bytes > 2 ** 32, rec.max_act_bytes
    assert "tail_chunk" in rec.extra


def _cover_hd_cascade(rec, convs):
    if HD_CASCADE_PAIRS == 8:
        tails = _tails(convs, 16)
        want = {f"{m}.conv{L}_{i}" for m in ("S", "cascade") for L in (5, 4) for i in (1, 2)}
        assert set(tails) == want, sorted(tails)
        assert "tail_chunk" in rec.extra
    assert any(r["op"] == "image_warp_concat" and (r["H"], r["W"]) == (1088, 1920) for r in rec.rows)


def _cover_kitti4(rec, convs):
    split = {r["H"] for r in convs if r["op"] == "conv3x3_split" and r["split_all"] and r["N"] == 8}
    assert {6, 12} <= split, split
    assert "chunk" in rec.extra


def _cover_tiny_bidir(rec, convs):
    _cover_tiny(rec, convs)
    assert "unswapped" in rec.extra


SHAPES = {   # run: (model class, pairs, H, W, image seed, coverage)
    "hd8": (network.MaskFlownetS, 8, 1080, 1920, 81, _cover_hd8),
    "hd_cascade": (network.MaskFlownet, HD_CASCADE_PAIRS, 1080, 1920, 82, _cover_hd_cascade),
    "kitti4": (network.MaskFlownetS, 4, 375, 1242, 83, _cover_kitti4),
    "tiny": (network.MaskFlownetS, 1, 64, 64, 84, _cover_tiny_bidir),
    "tiny_cascade": (network.MaskFlownet, 1, 64, 64, 85, _cover_tiny_cascade),
    "clip": (network.MaskFlownetS, 8, 436, 1024, 86, lambda rec, convs: None),   # 9 frames, as track_video calls it
}


def _inputs(run):
    cls, n, H, W, seed, _ = SHAPES[run]
    if run == "clip":
        x = _clip(seed, n + 1, H, W)
        return x[:n], x[1:]
    return _images_u8(seed=seed, n=n, h=H, w=W)


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(SHAPES))
@pytest.mark.usefixtures("fp64_references")
def test_every_launch_of_a_bidirectional_forward_against_float64(run, monkeypatch):
    cls, n, H, W, seed, cover = SHAPES[run]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    rec = BidirRecorder(monkeypatch, run, n)        # before the model packs anything
    model = _scaled_model(cls)
    u1, u2 = _inputs(run)
    fw, bw, occ_fw, occ_bw = network.predict_bidirectional(model, u1, u2)
    assert fw.shape == (n, H, W, 2) and bw.shape == (n, H, W, 2) and occ_fw.shape == (n, H, W)
    assert bool(torch.isfinite(fw).all()) and bool(torch.isfinite(bw).all())
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    rec.report()
    print(f"{run}: {len(rec.rows)} launches checked in {secs:.1f} s, peak {peak:.2f} GiB allocated, max |flow| "
          f"{float(torch.cat([fw, bw]).abs().max()):.3f} px")
    assert not rec.failures, "\n".join(rec.failures)

    # every convolution ran at batch 2N, as many as the graph has
    convs = [r for r in rec.rows if r["op"] in ("conv3x3_slices", "conv3x3_split")]
    assert len(convs) == _expected_convs("cascade" if cls is network.MaskFlownet else "fwd"), len(convs)
    assert {r["N"] for r in convs} == {2 * n}, sorted({r["N"] for r in convs})
    # pre- and post-processing, the consistency check, the occluded share of each direction
    PH, PW = ops.padded_size(H, W)
    pre = [r for r in rec.rows if r["op"] == "preprocess"]
    post = [r for r in rec.rows if r["op"] == "postprocess"]
    assert len(pre) == 1 and pre[0]["name"] == f"-> {PH}x{PW}" and len(post) == 1 and post[0]["N"] == 2 * n
    assert sum(r["op"] == "flow_consistency" for r in rec.rows) == 1
    assert all(0.0 < s < 1.0 for s in rec.occluded), rec.occluded
    # the wiring: every S-head correlation and warp, and the cascade's
    wires = set(rec.wiring)
    assert {f"S correlation L{L}: first operand is the pyramid output" for L in range(2, 7)} <= wires, sorted(wires)
    assert "S correlation L6: second operand is the pyramid output, halves swapped" in wires
    assert {f"S.deform{L}: warps the pyramid output, halves swapped" for L in range(2, 6)} <= wires, sorted(wires)
    assert "first pyramid launch reads the preprocess buffer in place" in wires
    if cls is network.MaskFlownet:
        assert {f"cascade correlation L{L}: first operand is the pyramid output" for L in range(2, 7)} <= wires
        assert {"image_warp_concat: im1 is the preprocess buffer", "image_warp_concat: im2 is im1, halves swapped"} | \
            {f"cascade.deform{L}: warps the unswapped pyramid output" for L in (2, 3)} | \
            {f"cascade.deform{L}: warps the pyramid output, halves swapped" for L in (4, 5, 6)} <= wires, sorted(wires)
    assert all(rec.wiring.values())
    # controls
    assert set(Recorder.KINDS) <= set(rec.controls), sorted(rec.controls)
    for tag, (name, rs) in rec.controls.items():
        assert min(rs.values()) >= CONTROL_MARGIN, (tag, name, rs)
    assert "unswapped" in rec.extra
    for tag, (name, r) in rec.extra.items():
        assert r >= CONTROL_MARGIN, (tag, name, r)
    differ, excluded, _ = rec.exchanged
    assert differ > 0 and differ >= CONTROL_MARGIN * excluded, rec.exchanged
    cover(rec, convs)


@pytest.mark.gpu
@pytest.mark.usefixtures("fp64_references")
def test_every_convolution_of_a_bf16_bidirectional_forward_against_float64(monkeypatch):
    """hd8 in bf16 mode: every convolution meets the bf16 bound of test_bf16_mode.py and ran the one-product variant."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    rec = BF16Recorder(monkeypatch, "hd8-bf16")
    model = _scaled_model(network.MaskFlownetS)
    model.inference_precision = "bf16"
    u1, u2 = _inputs("hd8")
    fw, bw, _, _ = network.predict_bidirectional(model, u1, u2)
    assert bool(torch.isfinite(fw).all()) and bool(torch.isfinite(bw).all())
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    rec.report()
    print(f"hd8-bf16: {len(rec.rows)} launches checked in {secs:.1f} s, peak {peak:.2f} GiB allocated")
    assert not rec.failures, "\n".join(rec.failures)
    convs = [r for r in rec.rows if r["op"] in ("conv3x3_slices", "conv3x3_split")]
    assert len(convs) == _expected_convs("fwd") and {r["N"] for r in convs} == {16}, len(convs)
    assert set(BF16Recorder.KINDS) <= set(rec.controls), sorted(rec.controls)
    for tag, (name, rs) in rec.controls.items():
        assert min(rs.values()) >= CONTROL_MARGIN, (tag, name, rs)
    assert {r["name"] for r in convs if r["ws"]} == {"S.conv5_1", "S.conv5_2", "S.conv4_1", "S.conv4_2"}


@pytest.mark.gpu
def test_bidirectional_video_predictor_graph_equals_eager_at_1080p():
    """VideoFlowPredictor(bidirectional=True) at the tools' batch of 8 on a 9-frame 1080p clip (one full batch): every
    output equals predict_bidirectional + ops.flow_to_color run eagerly, bit for bit, under deterministic algorithms."""
    model = _scaled_model(network.MaskFlownetS)
    x = _clip(87, 9, 1080, 1920)
    frames = x.permute(0, 2, 3, 1).contiguous().cpu().numpy()
    with _deterministic():
        pred = VideoFlowPredictor(model, batch=8, want_flow=True, bidirectional=True)
        got = list(pred.run(iter(frames)))
        fw, bw, occ_fw, occ_bw = network.predict_bidirectional(model, x[:8], x[1:])
        rgb, _ = ops.flow_to_color(fw)
        torch.cuda.synchronize()
    assert len(got) == 8
    occ = float(occ_fw.float().mean())
    assert 0.0 < occ < 1.0, occ
    for t in range(8):
        for g, e, nm in zip(got[t], (rgb, fw, bw, occ_fw, occ_bw), ("rgb", "flow", "flow_bw", "occ_fw", "occ_bw")):
            _same(torch.from_numpy(np.ascontiguousarray(g)), e[t].cpu(), f"pair {t} {nm}")
