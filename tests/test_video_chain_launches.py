"""Every launch of the video tools' chains (network.segment_motion, network.track_video, network.stabilize_video and
network.interpolate_frames) against float64, at the tools' default batch of 8 on 1080p frames, and which pair each frame
reads.

Each tool runs the bidirectional (or one-way) forward on batches of B pairs, the last batch padded with the last frame,
then its own kernels.  test_bidirectional_launches.py checks the forward launch by launch; the tools' kernels are checked
in their own files on synthetic flows.  Here ChainRecorder replaces the ops the chains call through the module
(ops.affine_motion, ops.segment_motion, ops.track_start / track_texture / track_advance / track_seed,
ops.warp_frames_affine, ops.interpolate_frames, ops.flow_consistency) and network._pair_flows, which every forward of
the chains and of network.predict_bidirectional goes through.  Each wrapper runs the original, synchronises, copies what
the launch read and wrote to the host and judges that launch alone against the oracle on the inputs it read, with the
judges the kernels' own files use, from launchcheck (the forward and the masks are logged for the wiring only):
  * affine_motion: stabilize._check_fit against stabilize_ref.fit (corners within 1e-6 px, residual within 1e-5 px
    plus one float32 ulp, NaN in the same places);
  * segment_motion: motion_segment._check against motionseg_ref.segment (labels, count, dropped, area, box,
    centroid and peak exact; dx, dy within the fixed-point bound);
  * track_texture bit for bit against track_ref.texture; track_advance with tracking._compare_advance (exclusions
    counted in a Tally, at most EXCLUDED_MAX) and track_seed with tracking._compare_seed (exact), both from the
    kernel's own previous state read out of the TrackState;
  * warp_frames_affine: stabilize._check_warp against stabilize_ref.warp; interpolate_frames: interpolate._check
    against interp_ref.interpolate.
Per-launch judging cannot see the wiring, because each launch is judged on whatever it read.  So the recorded flows,
masks, residuals and fits are indexed by global pair p = k0 + j (the real pairs j < nb of each batch only) and the
wiring is checked bit for bit: every fit and every pair of occlusion masks read the flows of its batch; every
segmentation read side a from its batch and side b from the backward rows shifted by one, row 0 from the previous
batch's last pair (NaN and 0 at k0 = 0); tracking and stabilisation compute no masks; the last frame reads pair P - 1's
backward side alone; advance k read pair k - 1's flows and frame k - 1's state; seed k read frame k's texture; the padded pairs are never advanced; queries are born in their frames; the
stabiliser's affine and ok rows are the fits of pairs 0..P-1, M is stabilize_ref.path of them within 1e-9 px at the
corners and the warp read the clip and M.  Segmentation is then restated with the batching removed: frame t takes side a
from pair t (t < P) and side b from pair t - 1 (t >= 1), through motionseg_ref.segment, and must equal the chain's
result.  Launch counts per kind must equal what the chain implies.

Runs (MaskFlownet-S and the cascade with random weights, flow heads scaled by FLOW_HEAD_SCALE so that both occlusion
decisions occur, under deterministic algorithms): hd, an 11-frame 1080x1920 clip at batch 8 (a full batch, then 2 real
pairs and 6 padded ones) through all three chains, and network.interpolate_frames on its first 8 pairs at times 0.25,
0.5 and 0.75; kitti, the cascade on an 8-frame 375x1242 clip at batch 3 (pairs 3 + 3 + 1, two carries); short, 64x64
clips of 2 and 1 frames (P = 1 and P = 0).  The network's flows follow nothing in the clip and stay below 2 px, so the
segmentation thresholds are the 0.9 and 0.99 quantiles of the first batch's finite forward residuals, from a pre-pass
outside the recorder, with MAX_OBJECTS = 4 (on an H100: hd 0.60 and 1.09 px, kitti 0.51 and 0.93 px, short 0.30 and
0.40 px).

Controls, on the real launches of hd: each judge must reject a changed rule (4-connectivity and max score for the
segmentation, weights never updated for the fit, the warp half a pixel off, the flow read at the rounded position for
every advance that starts from a TRACKED slot, seeding that ignores coverage, a dropped corner for the interpolation),
and each wrong wiring must disagree with the chain: side b from pair t, frame 0's side b as residual 0 (a carry never
reset), the last frame from pair P - 2, advance k against pair k's flows, seed k against frame k - 1's texture, the
camera path from fits shifted by one pair.  test_shared_chain_wiring_restatements_on_host runs the same recorder and
wiring checks on the CPU, with the oracles standing in for the kernels and hand-made per-pair flows, at B = 3 and P = 7:
the right assignment passes and every wiring control fails.

Not checked here: video denoising, whose chain (network.denoise_video, and VideoDenoiser's ring of frames and flows)
test_denoise_chain_launches.py checks launch by launch and wire by wire in the same way.
"""
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from maskflownet_b200 import network, ops
from oracle import interp_ref
from oracle import motionseg_ref as MR
from oracle import stabilize_ref as SR
from oracle import track_ref as TR

from launchcheck.inputs import _clip, _deterministic, _scaled_model
from launchcheck.interpolate import (EXCLUDED_MAX as INTERP_EXCLUDED_MAX, _check as _check_interp,
                                     _mismatch as _interp_mismatch)
from launchcheck.motion_segment import _check as _check_seg, _mismatch as _seg_mismatch
from launchcheck.stabilize import CORNER_TOL, WARP_EXACT, _check_fit, _check_warp, _fit_mismatch, _warp_mismatch
from launchcheck.tracking import Tally, _compare_advance, _compare_seed

OPS = ("affine_motion", "segment_motion", "track_start", "track_texture", "track_advance", "track_seed",
       "warp_frames_affine", "interpolate_frames", "flow_consistency")
KINDS = ("fit", "segment", "texture", "advance", "seed", "warp", "interp")
CONTROL_KINDS = ("fit", "segment", "advance", "seed", "warp", "interp")     # the texture is compared bit for bit
MAX_OBJECTS = 4
PATH_TOL = 1e-9                 # px at the corners: M and stabilize_ref.path are both float64
MOVED_MIN = 1e-3                # px: some fit must move the corners this far from the identity
SEG_VARIANTS = ("side b from pair t", "frame 0's side b residual 0", "last frame from pair P-2")
TRACK_VARIANTS = ("advance k against pair k", "seed k against frame k-1")
STAB_VARIANTS = ("fits shifted by one pair",)


def _sync():
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        torch.cuda.synchronize()


def _host(t):
    """A host copy (never a view: the state tensors change under it)."""
    if t is None:
        return None
    t = t.detach()
    return (t.cpu() if t.is_cuda else t.clone()).numpy()


def _eq(a, b):
    """Bit for bit (NaN equal to NaN), same shape and dtype."""
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


def _batches(P, B):
    return -(-P // B)


def _real_pairs(P, B):
    """(batch i, row j, global pair p = i B + j) of the real pairs."""
    return [(i, j, i * B + j) for i in range(_batches(P, B)) for j in range(min(B, P - i * B))]


def _seg_oracle(ins, kw, N, H, W, pool=map, control=None):
    """motionseg_ref.segment frame by frame; empty frames where neither side is given."""
    if all(t is None for t in ins):
        return (np.zeros((N, H, W), np.uint8), np.zeros((N, kw["max_objects"], 10)), np.zeros(N, np.int64),
                np.zeros(N, np.int64))
    outs = list(pool(lambda n: MR.segment(*(None if t is None else t[n:n + 1] for t in ins), control=control, **kw),
                     range(N)))
    return tuple(np.concatenate([o[k] for o in outs]) for k in range(4))


# ------------------------------------------------------------------------------------------------------------------
# the recorder: every launch judged on what it read, and the launches logged for the wiring
# ------------------------------------------------------------------------------------------------------------------
class ChainRecorder:
    """Wraps the ops and network entry points the chains call (`impl` replaces the originals: the host test passes the
    oracles).  self.log holds the current chain's launches (begin() starts a chain); self.judged counts the launches
    judged per kind; self.worst the worst figure per kind; self.ctl per kind the controls' (name, rejected, how far) on
    each launch (with controls=True)."""

    def __init__(self, monkeypatch, impl=None, controls=False, workers=None):
        self.orig = {n: getattr(ops, n) for n in OPS}
        self.orig.update(_pair_flows=network._pair_flows)
        self.orig.update(impl or {})
        for n in OPS:
            monkeypatch.setattr(ops, n, getattr(self, n))
        monkeypatch.setattr(network, "_pair_flows", self._pair_flows)
        self.controls = controls
        self.pool = ThreadPoolExecutor(workers or min(8, os.cpu_count() or 1))
        self.tally = Tally()
        self.judged = {k: 0 for k in KINDS}
        self.worst = dict(corner=0.0, residual=0.0, moved=0.0, warp_exact=1.0, interp_exact=1.0, interp_excluded=0,
                          interp_values=0)
        self.ctl = {k: [] for k in KINDS}
        self.begin()

    def begin(self):
        self.log = {k: [] for k in ("flows", "occ", "start") + KINDS}
        self.in_start = False

    def _map(self, fn, items):
        return self.pool.map(fn, items)

    # ---- the forwards and the occlusion masks ----------------------------------------------------------------------
    def _pair_flows(self, net, img1, img2, resize, bidirectional):
        flows = self.orig["_pair_flows"](net, img1, img2, resize, bidirectional)
        _sync()
        self.log["flows"].append(dict(flows=_host(flows), bidirectional=bidirectional))
        return flows

    def flow_consistency(self, flow_fw, flow_bw, alpha=0.01, beta=0.5):
        occ_fw, occ_bw = self.orig["flow_consistency"](flow_fw, flow_bw, alpha, beta)
        _sync()
        i = len(self.log["flows"]) - 1
        last = self.log["flows"][i]["flows"] if i >= 0 else None
        n = len(flow_fw)
        read = last is not None and _eq(_host(flow_fw), last[:n]) and _eq(_host(flow_bw), last[n:])
        self.log["occ"].append(dict(occ_fw=_host(occ_fw), occ_bw=_host(occ_bw), flows=i if read else None))
        return occ_fw, occ_bw

    # ---- stabilisation and segmentation ---------------------------------------------------------------------------
    def affine_motion(self, flow, iterations=ops.AFFINE_ITERATIONS, sigma=ops.AFFINE_SIGMA, want_residual=False):
        res = self.orig["affine_motion"](flow, iterations, sigma, want_residual)
        _sync()
        f = _host(flow)
        A, ok = _host(res[0]), _host(res[1])
        r = _host(res[2]) if want_residual else None
        N, H, W, _ = f.shape
        refs = list(self._map(lambda n: SR.fit(f[n:n + 1], iterations, sigma), range(N)))
        ref = tuple(np.concatenate([x[k] for x in refs]) for k in range(3))
        what = f"affine_motion launch {len(self.log['fit'])} ({N}x{H}x{W})"
        d = _check_fit((A, ok, r), ref, H, W, what)
        self.judged["fit"] += 1
        self.worst["corner"] = max(self.worst["corner"], d)
        if r is not None:
            both = ~np.isnan(r) & ~np.isnan(ref[2])
            self.worst["residual"] = max(self.worst["residual"], float(np.abs(r - ref[2])[both].max(initial=0.0)))
        moved = np.abs(SR.corners(A, H, W) - SR.corners(np.eye(2, 3), H, W)).max(initial=0.0)
        self.worst["moved"] = max(self.worst["moved"], float(moved))
        if self.controls:
            c = "no_reweight"
            dc, okbad, resbad = _fit_mismatch((A[:1], ok[:1], None if r is None else r[:1]),
                                              SR.fit(f[:1], iterations, sigma, control=c), H, W)
            self.ctl["fit"].append((c, dc > CORNER_TOL or okbad or resbad > 0, dc / CORNER_TOL))
        self.log["fit"].append(dict(flow=f, A=A, ok=ok, res=r))
        return res

    def segment_motion(self, res_a=None, occ_a=None, res_b=None, occ_b=None, flow_a=None, affine_a=None,
                       tau_lo=ops.SEG_TAU_LO, tau_hi=ops.SEG_TAU_HI, min_area=ops.SEG_MIN_AREA,
                       max_objects=ops.SEG_MAX_OBJECTS, shape=None):
        out = self.orig["segment_motion"](res_a, occ_a, res_b, occ_b, flow_a, affine_a, tau_lo, tau_hi, min_area,
                                          max_objects, shape)
        _sync()
        ins = tuple(_host(t) for t in (res_a, occ_a, res_b, occ_b, flow_a, affine_a))
        got = tuple(_host(t) for t in out)
        kw = dict(tau_lo=tau_lo, tau_hi=tau_hi, min_area=min_area, max_objects=max_objects)
        N, H, W = got[0].shape
        _check_seg(got, _seg_oracle(ins, kw, N, H, W, self._map), H, W,
                   f"segment_motion launch {len(self.log['segment'])}")
        self.judged["segment"] += 1
        if self.controls and ins[0] is not None and ins[2] is not None:
            for c in MR.CONTROLS:
                ref = _seg_oracle(ins, kw, N, H, W, self._map, control=c)
                far = int((got[0] != ref[0]).sum()) + int((np.asarray(got[2]) != ref[2]).sum())
                self.ctl["segment"].append((c, _seg_mismatch(got, ref, H, W) is not None, far))
        self.log["segment"].append(dict(ins=ins, got=got, kw=kw))
        return out

    def warp_frames_affine(self, frames, M):
        out = self.orig["warp_frames_affine"](frames, M)
        _sync()
        src, Mh, got = _host(frames), _host(M), _host(out)
        ref = np.concatenate(list(self._map(lambda n: SR.warp(src[n:n + 1], Mh[n:n + 1]), range(len(src)))))
        e = _check_warp(got, ref, f"warp_frames_affine launch {len(self.log['warp'])}")
        self.judged["warp"] += 1
        self.worst["warp_exact"] = min(self.worst["warp_exact"], e)
        if self.controls:
            c = "warp_half_pixel"
            ctl = np.concatenate(list(self._map(lambda n: SR.warp(src[n:n + 1], Mh[n:n + 1], control=c),
                                                range(len(src)))))
            dmax, exact = _warp_mismatch(got, ctl)
            self.ctl["warp"].append((c, dmax > 1 or exact < WARP_EXACT, 1.0 - exact))
        self.log["warp"].append(dict(frames=src, M=Mh, out=got))
        return out

    # ---- tracking ---------------------------------------------------------------------------------------------------
    def track_start(self, state, frame, out_xy=None, out_status=None, out_dropped=None):
        self.in_start = True          # its texture and seed launches go through the wrappers below
        try:
            res = self.orig["track_start"](state, frame, out_xy, out_status, out_dropped)
        finally:
            self.in_start = False
        self.log["start"].append(_host(frame))
        return res

    def track_texture(self, frames, spacing=8):
        lam, lmax = self.orig["track_texture"](frames, spacing)
        _sync()
        f = _host(frames)
        f4 = f if f.ndim == 4 else f[None]
        L = _host(lam)
        L3 = L if L.ndim == 3 else L[None]
        M = _host(lmax)
        refs = list(self._map(lambda n: TR.texture(f4[n], spacing), range(len(f4))))
        for n, ref in enumerate(refs):
            assert np.array_equal(L3[n], ref) and M[n] == ref.max(initial=0.0), \
                f"track_texture launch {len(self.log['texture'])} frame {n}"
        self.judged["texture"] += 1
        self.log["texture"].append(dict(frames=f4, lam=L3, lmax=M, start=self.in_start))
        return lam, lmax

    def track_advance(self, state, flow_fw, flow_bw):
        _sync()
        prev_pos, prev_status = _host(state.pos), _host(state.status)
        self.orig["track_advance"](state, flow_fw, flow_bw)
        _sync()
        pos, status = _host(state.pos), _host(state.status)
        fw, bw = _host(flow_fw), _host(flow_bw)
        k = len(self.log["advance"]) + 1
        bad = _compare_advance(prev_pos, prev_status, pos, status, fw, bw, self.tally)
        assert bad == 0, f"track_advance {k}: {bad} slots differ from the oracle"
        self.judged["advance"] += 1
        # seeds lie on whole pixels, where the rounded read is the bilinear one; a TRACKED slot has moved off them
        if self.controls and (prev_status == TR.TRACKED).any():
            c = "sample_rounded"
            far = _compare_advance(prev_pos, prev_status, pos, status, fw, bw, None, control=c)
            self.ctl["advance"].append((c, far > 0, far))
        self.log["advance"].append(dict(fw=fw, bw=bw, prev_pos=prev_pos, prev_status=prev_status))

    def track_seed(self, state, lambda2, lambda_max, out_xy=None, out_status=None, out_dropped=None):
        _sync()
        adv_pos, adv_status, frame = _host(state.pos), _host(state.status), int(state.frame.item())
        xy, st, dropped = self.orig["track_seed"](state, lambda2, lambda_max, out_xy, out_status, out_dropped)
        _sync()
        lam, lmax, q = _host(lambda2), _host(lambda_max), _host(state.queries)
        gxy, gst, gd = _host(xy), _host(st), int(_host(dropped).reshape(-1)[0])
        args = (adv_pos, adv_status, lam, lmax, q, frame, state.spacing, state.tau, state.H, state.W, gxy, gst, gd)
        bad = _compare_seed(*args)
        assert bad == 0, f"track_seed of frame {frame}: {bad} slots or the dropped count differ from the oracle"
        self.judged["seed"] += 1
        if self.controls and frame >= 1:
            c = "ignore_coverage"
            far = _compare_seed(*args, control=c)
            self.ctl["seed"].append((c, far > 0, far))
        self.log["seed"].append(dict(lam=lam, lmax=lmax, frame=frame, start=self.in_start))
        return xy, st, dropped

    # ---- interpolation ----------------------------------------------------------------------------------------------
    def interpolate_frames(self, img0, img1, flow_fw, flow_bw, occ_fw, occ_bw, times, occ_weight=0.01):
        out = self.orig["interpolate_frames"](img0, img1, flow_fw, flow_bw, occ_fw, occ_bw, times, occ_weight)
        _sync()
        a = [_host(t) for t in (img0, img1, flow_fw, flow_bw, occ_fw, occ_bw)]
        got = _host(out)
        assert got.ndim == 5, got.shape
        ts = ops._interp_times(times, "interpolate_frames")

        def one(n, control=None):
            s = [v[n:n + 1] for v in a]
            return s, interp_ref.interpolate(*s, ts, occ_weight, control=control)

        excl = total = exact = 0
        for n, (s, ref) in enumerate(self._map(one, range(len(got)))):
            e, t = _check_interp(got[n:n + 1], ref, s[0], s[1], ts, f"interpolate_frames pair {n}")
            excl, total, exact = excl + e, total + t, exact + int((got[n:n + 1] == ref["frames"]).sum())
        assert excl <= INTERP_EXCLUDED_MAX * total, (excl, total)
        self.judged["interp"] += 1
        self.worst["interp_exact"] = min(self.worst["interp_exact"], exact / total)
        self.worst["interp_excluded"] += excl
        self.worst["interp_values"] += total
        if self.controls:
            c = "drop_corner"
            s, ref = one(0, c)
            bad, _, t, _ = _interp_mismatch(got[:1], ref, s[0], s[1], ts)
            self.ctl["interp"].append((c, bad > 0, bad / t))
        self.log["interp"].append(1)
        return out


# ------------------------------------------------------------------------------------------------------------------
# the wiring, from the logs of one chain (wrong assignments as `variant`, for the controls)
# ------------------------------------------------------------------------------------------------------------------
def _seg_pairs(log, B, P):
    """Per global pair p: its forward and backward flows, masks, residuals and forward fit, from the batch launches."""
    pairs = []
    for i, j, p in _real_pairs(P, B):
        occ, fit = log["occ"][i], log["fit"][i]
        pairs.append(dict(fw=log["flows"][i]["flows"][j], ofw=occ["occ_fw"][j], obw=occ["occ_bw"][j],
                          res_fw=fit["res"][j], A_fw=fit["A"][j], res_bw=fit["res"][B + j]))
    return pairs


def _seg_wiring(log, B, P, H, W):
    n = _batches(P, B)
    w = {"launches: ceil(P/B) forwards and fits, ceil(P/B) + 1 segmentations":
         len(log["flows"]) == n and all(f["bidirectional"] for f in log["flows"]) and len(log["occ"]) == n and
         len(log["fit"]) == n and len(log["segment"]) == n + 1}
    if not all(w.values()):
        return w
    for i in range(n):
        fw, bw = log["flows"][i]["flows"][:B], log["flows"][i]["flows"][B:]
        ofw, obw = log["occ"][i]["occ_fw"], log["occ"][i]["occ_bw"]
        fit, (res_a, occ_a, res_b, occ_b, flow_a, affine_a) = log["fit"][i], log["segment"][i]["ins"]
        w[f"masks {i} read flow_fw and flow_bw of forward {i}"] = log["occ"][i]["flows"] == i
        w[f"fit {i} read cat(flow_fw, flow_bw)"] = _eq(fit["flow"], np.concatenate([fw, bw]))
        w[f"segment {i} side a: residual rows [0, B), occ_fw, flow_fw, affine[:B]"] = \
            _eq(res_a, fit["res"][:B]) and _eq(occ_a, ofw) and _eq(flow_a, fw) and _eq(affine_a, fit["A"][:B])
        if i == 0:
            carry = np.full((1, H, W), np.nan, np.float32), np.zeros((1, H, W), np.uint8)
        else:
            carry = log["fit"][i - 1]["res"][2 * B - 1:], log["occ"][i - 1]["occ_bw"][B - 1:]
        w[f"segment {i} side b row 0: pair k0 - 1's backward residual and mask (NaN and 0 at k0 = 0)"] = \
            _eq(res_b[:1], carry[0]) and _eq(occ_b[:1], carry[1])
        w[f"segment {i} side b rows 1..B-1: backward rows 0..B-2"] = \
            _eq(res_b[1:], fit["res"][B:2 * B - 1]) and _eq(occ_b[1:], obw[:B - 1])
    last = log["segment"][-1]["ins"]
    if P == 0:
        w["one empty frame"] = all(t is None for t in last)
    else:
        i, nb = n - 1, P - (n - 1) * B
        w["last frame: pair P - 1's backward residual and mask alone"] = \
            all(last[k] is None for k in (0, 1, 4, 5)) and _eq(last[2], log["fit"][i]["res"][B + nb - 1:B + nb]) and \
            _eq(last[3], log["occ"][i]["occ_bw"][nb - 1:nb])
    return w


def _seg_restate(pairs, T, kw, H, W, pool=map, variant=None):
    """The segmentation without the batching: frame t takes side a from pair t (t < P) and side b from pair t - 1
    (t >= 1), or the sides `variant` names."""
    P = T - 1

    def frame(t):
        a = t if t < P else None
        b = t - 1 if t >= 1 else None
        if variant == "side b from pair t":
            b = t if t < P else None
        if variant == "last frame from pair P-2" and t == P:
            b = P - 2 if P >= 2 else None
        ra = oa = fa = Aa = rb = ob = None
        if a is not None:
            ra, oa, fa, Aa = (pairs[a][k][None] for k in ("res_fw", "ofw", "fw", "A_fw"))
        if variant == "frame 0's side b residual 0" and t == 0:
            rb, ob = np.zeros((1, H, W), np.float32), np.zeros((1, H, W), np.uint8)
        elif b is not None:
            rb, ob = pairs[b]["res_bw"][None], pairs[b]["obw"][None]
        return _seg_oracle((ra, oa, rb, ob, fa, Aa), kw, 1, H, W)

    outs = list(pool(frame, range(T)))
    return tuple(np.concatenate([o[k] for o in outs]) for k in range(4))


def _track_wiring(log, B, P, clip, result, queries, spacing, variant=None):
    xy, status, _ = result
    n = _batches(P, B)
    tex = [t for t in log["texture"] if not t["start"]]
    seeds = [s for s in log["seed"] if not s["start"]]
    starts = [s for s in log["seed"] if s["start"]]
    w = {"launches: ceil(P/B) forwards and textures, P advances, P seeds (and the start's texture and seed)":
         len(log["flows"]) == n and all(f["bidirectional"] for f in log["flows"]) and not log["occ"] and
         len(tex) == n and len(log["advance"]) == P and len(seeds) == P and len(log["start"]) == 1 and
         len(starts) == 1 and len(log["texture"]) == n + 1}
    if not all(w.values()):
        return w
    fl = [f["flows"] for f in log["flows"]]
    pairs = {p: (fl[i][j], fl[i][B + j]) for i, j, p in _real_pairs(P, B)}
    padded = [(fl[i][j], fl[i][B + j]) for i in range(n) for j in range(min(B, P - i * B), B)]
    ref0 = TR.texture(clip[0], spacing)
    w["start: frame 0's texture, frame counter 0"] = _eq(log["start"][0], clip[0]) and starts[0]["frame"] == 0 and \
        np.array_equal(starts[0]["lam"], ref0) and starts[0]["lmax"][0] == ref0.max(initial=0.0)
    for k in range(1, P + 1):
        adv, sd = log["advance"][k - 1], seeds[k - 1]
        src = k if variant == "advance k against pair k" else k - 1
        w[f"advance {k} read pair {k - 1}'s flow_fw and flow_bw"] = \
            src in pairs and _eq(adv["fw"], pairs[src][0]) and _eq(adv["bw"], pairs[src][1])
        w[f"advance {k} started from frame {k - 1}'s xy and status"] = \
            _eq(adv["prev_pos"], xy[k - 1]) and _eq(adv["prev_status"], status[k - 1])
        w[f"advance {k} read no padded pair"] = not any(_eq(adv["fw"], f) or _eq(adv["bw"], b) for f, b in padded)
        f = k - 1 if variant == "seed k against frame k-1" else k
        ref = TR.texture(clip[f], spacing)
        w[f"seed {k}: frame {k}'s texture, frame counter {k}"] = sd["frame"] == k and \
            np.array_equal(sd["lam"], ref) and sd["lmax"][0] == ref.max(initial=0.0)
    for m, (t, x, y) in enumerate(queries):
        t = int(t)
        if t <= P and 0 <= x <= clip.shape[2] - 1 and 0 <= y <= clip.shape[1] - 1:
            w[f"query {m} born in frame {t}"] = status[t, m] == TR.BORN and bool((status[:t, m] == TR.EMPTY).all()) \
                and np.array_equal(xy[t, m], np.array([x, y], np.float32))
    return w


def _stab_wiring(log, B, P, clip, result, radius, crop, variant=None):
    """(wiring, corner distance between M and stabilize_ref.path of the returned fits)."""
    out, affine, ok, M = result
    H, W = clip.shape[1:3]
    n = _batches(P, B)
    w = {"launches: ceil(P/B) forwards and fits, one warp":
         len(log["flows"]) == n and not any(f["bidirectional"] for f in log["flows"]) and not log["occ"] and
         len(log["fit"]) == n and len(log["warp"]) == 1}
    if not all(w.values()):
        return w, float("inf")
    for i in range(n):
        w[f"fit {i} read forward {i}'s flow"] = _eq(log["fit"][i]["flow"], log["flows"][i]["flows"])
    w["affine and ok rows are the fits of pairs 0..P-1"] = len(affine) == P and all(
        _eq(affine[p], log["fit"][i]["A"][j]) and ok[p] == log["fit"][i]["ok"][j] for i, j, p in _real_pairs(P, B))
    A, g = affine, ok
    if variant == "fits shifted by one pair":
        A, g = np.concatenate([np.eye(2, 3)[None], affine[:-1]]), np.concatenate([[True], ok[:-1]])
    d = float(np.abs(SR.corners(M, H, W) - SR.corners(SR.path(A, g, H, W, radius, crop), H, W)).max())
    w["M is stabilize_ref.path of the fits"] = d <= PATH_TOL
    warp = log["warp"][0]
    w["the warp read the clip and M, and its output is returned"] = \
        _eq(warp["frames"], clip) and _eq(warp["M"], M) and _eq(warp["out"], out)
    return w, d


# ------------------------------------------------------------------------------------------------------------------
# one run of the three chains through the recorder
# ------------------------------------------------------------------------------------------------------------------
def _queries(B, P, H, W):
    """Queries born in frames 0, B, B + 1 and P at fractional positions inside the frame, and four at frame 0 in the
    frame's corners."""
    q = [[t, (0.3 + 0.1 * m) * W + 0.25, (0.4 + 0.1 * m) * H + 0.5] for m, t in enumerate((0, B, B + 1, P))]
    q += [[0, x, y] for x in (0, W - 1) for y in (0, H - 1)]
    return np.array(q, np.float32)


def _run_chains(rec, model, clip, B, kw, pool, spacing=8, radius=15, crop=0.9):
    """Runs the three chains on `clip` (T,H,W,3) uint8 through the recorder and checks their wiring.  Returns a dict
    per chain of (result, wiring) and what the controls need."""
    T, H, W, _ = clip.shape
    P = T - 1
    host_clip = _host(clip)
    out = {}

    rec.begin()
    seg = [_host(t) for t in network.segment_motion(model, clip, batch=B, **kw)]
    w = _seg_wiring(rec.log, B, P, H, W)
    pairs = _seg_pairs(rec.log, B, P) if all(w.values()) else None
    if pairs is not None:
        _check_seg(seg, _seg_restate(pairs, T, kw, H, W, pool), H, W, "segmentation restated without the batching")
    out["segment"] = dict(result=seg, wiring=w, pairs=pairs, log=rec.log)

    rec.begin()
    q = _queries(B, P, H, W)
    trk = [_host(t) for t in network.track_video(model, clip, batch=B, spacing=spacing, queries=q)]
    out["track"] = dict(result=trk, wiring=_track_wiring(rec.log, B, P, host_clip, trk, q, spacing), queries=q,
                        log=rec.log)

    rec.begin()
    res = network.stabilize_video(model, clip, batch=B, radius=radius, crop=crop)
    stab = [_host(t) for t in res[:3]] + [res[3]]
    w, d = _stab_wiring(rec.log, B, P, host_clip, stab, radius, crop)
    out["stab"] = dict(result=stab, wiring=w, path_d=d, log=rec.log)
    return out


def _wiring_controls(runs, B, H, W, kw, pool, spacing=8, radius=15, crop=0.9):
    """For each wrong assignment: how far it disagrees with the chain (frames, checks or px; 0 = it agrees)."""
    far = {}
    seg, trk, stab = runs["segment"], runs["track"], runs["stab"]
    T = len(seg["result"][0])
    for v in SEG_VARIANTS:
        ref = _seg_restate(seg["pairs"], T, kw, H, W, pool, v)
        far[v] = int(sum(_seg_mismatch([x[t:t + 1] for x in seg["result"]], [x[t:t + 1] for x in ref], H, W)
                         is not None for t in range(T)))
    clip = stab["log"]["warp"][0]["frames"]
    for v in TRACK_VARIANTS:
        w = _track_wiring(trk["log"], B, T - 1, clip, trk["result"], trk["queries"], spacing, v)
        far[v] = sum(not ok for ok in w.values())
    for v in STAB_VARIANTS:
        far[v] = _stab_wiring(stab["log"], B, T - 1, clip, stab["result"], radius, crop, v)[1]
    return far


# ------------------------------------------------------------------------------------------------------------------
# CPU: the recorder and the wiring checks with the oracles standing in for the kernels
# ------------------------------------------------------------------------------------------------------------------
HB, HP, HH, HW = 3, 7, 24, 32          # batch, pairs, frame size of the host test
HOST_KW = dict(tau_lo=1.0, tau_hi=2.0, min_area=4, max_objects=MAX_OBJECTS)


def _hand_flow(i, j, H, W):
    """The flow a fake forward gives from frame i to frame j: a small random camera motion with 0.1 px noise, drawn per
    pair (padded pairs (P, P) included), and a 6 x 6 block moving 3-5 px against it, in frame i's place for the block,
    so that both directions of a frame see it there."""
    rng = np.random.default_rng(1000 * i + j)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    L = np.eye(2) + rng.uniform(-0.02, 0.02, (2, 2))
    t = rng.uniform(-1, 1, 2)
    f = np.stack([L[0, 0] * x + L[0, 1] * y + t[0] - x, L[1, 0] * x + L[1, 1] * y + t[1] - y], -1)
    f += rng.normal(0, 0.1, f.shape)
    y0, x0 = np.random.default_rng(i).integers(2, (H - 8, W - 8))
    f[y0:y0 + 6, x0:x0 + 6] += rng.uniform(3, 5, 2) * rng.choice([-1, 1], 2)
    return f.astype(np.float32)


def _hand_occ(i, j, H, W):
    return (np.random.default_rng(7000 + 1000 * i + j).random((H, W)) < 0.05).astype(np.uint8)


def _host_impl():
    """The chains' device steps on the host: per-pair flows from _hand_flow (frame t carries t in its first byte) and
    the oracles for the kernels."""
    T = torch.from_numpy

    def ids(a, b):
        return [(int(u[0, 0, 0]), int(v[0, 0, 0])) for u, v in zip(a, b)]

    served = {}          # the pair ids of each flow tensor _pair_flows returned, by its data pointer

    def _pair_flows(net, img1, img2, resize, bidirectional):
        H, W = img1.shape[2:]
        p = ids(img1, img2)
        flows = T(np.stack([_hand_flow(*(ij[::-1] if rev else ij), H, W)
                            for rev in ((False, True) if bidirectional else (False,)) for ij in p]))
        served[flows.data_ptr()] = p
        return flows

    def flow_consistency(flow_fw, flow_bw, alpha=0.01, beta=0.5):
        H, W = flow_fw.shape[1:3]
        p = served[flow_fw.data_ptr()]
        return tuple(T(np.stack([_hand_occ(*(ij[::-1] if rev else ij), H, W) for ij in p])) for rev in (False, True))

    def affine_motion(flow, iterations=ops.AFFINE_ITERATIONS, sigma=ops.AFFINE_SIGMA, want_residual=False):
        A, ok, r = SR.fit(flow.numpy(), iterations, sigma)
        return (T(A), T(ok), T(r)) if want_residual else (T(A), T(ok))

    def segment_motion(res_a=None, occ_a=None, res_b=None, occ_b=None, flow_a=None, affine_a=None, tau_lo=1.0,
                       tau_hi=2.0, min_area=64, max_objects=255, shape=None):
        ins = tuple(_host(t) for t in (res_a, occ_a, res_b, occ_b, flow_a, affine_a))
        N, H, W = shape if shape is not None else next(t for t in ins if t is not None).shape[:3]
        out = _seg_oracle(ins, dict(tau_lo=tau_lo, tau_hi=tau_hi, min_area=min_area, max_objects=max_objects), N, H, W)
        return T(out[0]), T(out[1]), T(out[2].astype(np.int32)), T(out[3].astype(np.int32))

    def track_texture(frames, spacing=8):
        f = frames.numpy()
        f4 = f if f.ndim == 4 else f[None]
        lam = np.stack([TR.texture(x, spacing) for x in f4])
        lmax = lam.reshape(len(f4), -1).max(1, initial=0.0)
        return (T(lam), T(lmax)) if f.ndim == 4 else (T(lam[0]), T(lmax))

    def track_advance(state, flow_fw, flow_bw):
        a = TR.advance(state.pos.numpy(), state.status.numpy(), flow_fw.numpy(), flow_bw.numpy(), state.alpha,
                       state.beta, state.boundary)
        state.pos.copy_(T(a["pos"]))
        state.status.copy_(T(a["status"]))

    def track_seed(state, lambda2, lambda_max, out_xy=None, out_status=None, out_dropped=None):
        pos, st, d = TR.seed(state.pos.numpy(), state.status.numpy(), lambda2.numpy(), lambda_max.numpy(),
                             state.queries.numpy(), int(state.frame.item()), state.spacing, state.tau, state.H, state.W)
        state.pos.copy_(T(pos))
        state.status.copy_(T(st))
        state.frame += 1
        xy = torch.empty((state.K, 2)) if out_xy is None else out_xy
        s = torch.empty((state.K,), dtype=torch.uint8) if out_status is None else out_status
        dropped = state.dropped if out_dropped is None else out_dropped
        xy.copy_(T(pos))
        s.copy_(T(st))
        dropped.fill_(int(d))
        return xy, s, dropped

    def warp_frames_affine(frames, M):
        return T(SR.warp(frames.numpy(), M.numpy()))

    return dict(_pair_flows=_pair_flows, flow_consistency=flow_consistency, affine_motion=affine_motion,
                segment_motion=segment_motion, track_texture=track_texture, track_advance=track_advance,
                track_seed=track_seed, warp_frames_affine=warp_frames_affine)


def _hand_clip(T, H, W):
    rng = np.random.default_rng(17)
    clip = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
    clip[:, 0, 0, 0] = np.arange(T)
    return torch.from_numpy(clip)


def test_shared_chain_wiring_restatements_on_host(monkeypatch):
    """B = 3, P = 7 (pairs 3 + 3 + 1, two carries): the chains run on the host with the oracles as their kernels; the
    wiring checks and the batch-free restatement pass, launch counts are the chain's, and every wrong assignment
    disagrees with the chain."""
    clip = _hand_clip(HP + 1, HH, HW)
    rec = ChainRecorder(monkeypatch, impl=_host_impl(), workers=1)
    runs = _run_chains(rec, None, clip, HB, HOST_KW, map, spacing=4, radius=2)
    monkeypatch.undo()
    for chain, r in runs.items():
        assert r["wiring"] and all(r["wiring"].values()), (chain, [k for k, ok in r["wiring"].items() if not ok])
    assert runs["stab"]["path_d"] <= PATH_TOL
    n = _batches(HP, HB)
    assert rec.judged == dict(fit=2 * n, segment=n + 1, texture=n + 1, advance=HP, seed=HP + 1, warp=1, interp=0)
    seg = runs["segment"]["result"]
    assert seg[2][0] >= 1 and seg[2].sum() >= HP, seg[2]        # frame 0 has an object: the carry control can see it
    far = _wiring_controls(runs, HB, HH, HW, HOST_KW, map, spacing=4, radius=2)
    print("wiring controls (frames / checks / px):", far)
    assert all(v > 0 for v in far.values()), far
    assert far["fits shifted by one pair"] > 1e3 * PATH_TOL


# ------------------------------------------------------------------------------------------------------------------
# GPU: the runs
# ------------------------------------------------------------------------------------------------------------------
RUNS = {   # run: (model class, batch, clip lengths, H, W, image seed, interpolate the first batch)
    "hd": (network.MaskFlownetS, 8, (11,), 1080, 1920, 91, True),
    "kitti": (network.MaskFlownet, 3, (8,), 375, 1242, 92, False),
    "short": (network.MaskFlownetS, 8, (2, 1), 64, 64, 93, False),
}


def _thresholds(model, clip, B):
    """tau_lo, tau_hi: the 0.9 and 0.99 quantiles of the finite forward residuals of the chain's first batch."""
    P = clip.shape[0] - 1
    x = clip[[min(j, P) for j in range(B + 1)]].permute(0, 3, 1, 2).contiguous()
    fw, bw, _, _ = network.predict_bidirectional(model, x[:B], x[1:])
    _, _, res = ops.affine_motion(torch.cat([fw, bw]), want_residual=True)
    r = _host(res[:B])
    lo, hi = np.quantile(r[np.isfinite(r)], [0.9, 0.99])
    return dict(tau_lo=float(lo), tau_hi=float(hi), max_objects=MAX_OBJECTS)


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
def test_every_launch_of_the_shared_video_chains_against_float64(run, monkeypatch):
    cls, B, lengths, H, W, seed, interp = RUNS[run]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    model = _scaled_model(cls)
    clips = [_clip(seed + T, T, H, W).permute(0, 2, 3, 1).contiguous() for T in lengths]
    with _deterministic():
        kw = _thresholds(model, clips[0], B)
        rec = ChainRecorder(monkeypatch, controls=run == "hd")
        runs = [_run_chains(rec, model, clip, B, kw, rec._map) for clip in clips]
        if interp:
            x = clips[0][:B + 1].permute(0, 3, 1, 2).contiguous()
            rec.begin()
            frames = network.interpolate_frames(model, x[:B], x[1:], (0.25, 0.5, 0.75))
            assert frames.shape == (B, 3, H, W, 3) and len(rec.log["flows"]) == 1 and rec.log["occ"][0]["flows"] == 0 \
                and rec.judged["interp"] == 1
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()

    # the launches judged per kind: what the chains imply
    want = dict.fromkeys(KINDS, 0)
    for T in lengths:
        P, n = T - 1, _batches(T - 1, B)
        want["fit"] += 2 * n
        want["segment"] += n + 1
        want["texture"] += n + 1          # one per batch and the start's
        want["advance"] += P
        want["seed"] += P + 1             # one per pair and the start's
        want["warp"] += 1
    want["interp"] = int(interp)
    w = rec.worst
    print(f"{run}: tau_lo {kw['tau_lo']:.4f} tau_hi {kw['tau_hi']:.4f} px; launches judged {rec.judged}")
    print(f"{run}: worst fit corner distance {w['corner']:.2e} px (bound {CORNER_TOL:g}), residual error "
          f"{w['residual']:.2e} px, largest corner motion {w['moved']:.3f} px; tracking excluded {rec.tally.excluded} "
          f"of {rec.tally.compared}; warp {100 * w['warp_exact']:.4f} % exact; interpolation "
          f"{100 * w['interp_exact']:.4f} % exact, {w['interp_excluded']} of {w['interp_values']} excluded")
    for r, T in zip(runs, lengths):
        seg, trk, stab = r["segment"]["result"], r["track"]["result"], r["stab"]
        print(f"{run} T={T}: objects per frame {seg[2].tolist()}, dropped {seg[3].tolist()}; track statuses "
              f"{np.bincount(trk[1].ravel(), minlength=6).tolist()}; M against stabilize_ref.path "
              f"{stab['path_d']:.2e} px")
        for chain in ("segment", "track", "stab"):
            bad = [k for k, ok in r[chain]["wiring"].items() if not ok]
            print(f"{run} T={T} {chain}: {len(r[chain]['wiring'])} wiring checks, {len(bad)} failed {bad}")
    print(f"{run}: {secs:.1f} s, peak {peak:.2f} GiB allocated")

    assert rec.judged == want, (rec.judged, want)
    rec.tally.check()
    for r in runs:
        for chain in ("segment", "track", "stab"):
            assert all(r[chain]["wiring"].values()), (chain, [k for k, ok in r[chain]["wiring"].items() if not ok])
        assert r["stab"]["path_d"] <= PATH_TOL

    if run in ("hd", "kitti"):
        seg, (xy, st, _), r = runs[0]["segment"]["result"], runs[0]["track"]["result"], runs[0]
        M = len(r["track"]["queries"])
        assert seg[2][0] >= 1 and (seg[3] > 0).any(), (seg[2], seg[3])
        assert set(np.unique(st).tolist()) == {TR.EMPTY, TR.TRACKED, TR.BORN, TR.LEFT, TR.OCCLUDED, TR.BOUNDARY}
        assert (st[1:, M:] == TR.BORN).any()                           # a dense slot seeded after frame 0
        assert w["moved"] >= MOVED_MIN, w["moved"]

    if run == "hd":
        for kind in CONTROL_KINDS:
            ctl = rec.ctl[kind]
            print(f"hd control {kind}: " + ", ".join(f"{c} {'rejected' if ok else 'PASSED'} ({far:.3g})"
                                                      for c, ok, far in ctl))
            assert ctl and all(ok for _, ok, _ in ctl), (kind, ctl)
        assert {c for c, _, _ in rec.ctl["segment"]} == set(MR.CONTROLS)
        far = _wiring_controls(runs[0], B, H, W, kw, rec._map)
        print("hd wiring controls (frames / checks / px):", far)
        assert all(v > 0 for v in far.values()), far
        assert far["fits shifted by one pair"] > PATH_TOL, far
    rec.pool.shutdown()
