"""Every launch of the video denoising chain (network.denoise_video and video.VideoDenoiser) against float64 at the video
tools' sizes, on the flows the networks produce, and which frames and flows each launch reads.

test_denoise.py checks the kernels against oracle/denoise_ref.py on synthetic flows, and VideoDenoiser against
network.denoise_video bit for bit at 100x150; both paths share network._frame_pair_flows, so a wrong pair index or a
swapped direction in what both store would pass there.  Here DenoiseRecorder wraps network._pair_flows (each batch's 2B
flows, the rows named by the clip frames they read: real pair p = k0 + j, or a padded pair of the last frame with
itself), ops.denoise_frames, ops.estimate_noise (ops.median_noise looks it up in the module, so both are caught),
video._FrameRing._store (which ring, which slots and which frame or pair indices each copy writes) and torch.cuda.Event
(every record and wait, with its stream, in host order).  Each wrapper runs the original, synchronises, copies what the
launch read and wrote to the host and judges that launch alone: denoise_frames against denoise_ref.denoise on the ring
arrays exactly as the launch read them, with its own t0, n, t_lo, t_hi, radius, sigma, h, patch, alpha and beta, frame
by frame (launchcheck.denoise._check with flipped=FLIPPED: test_denoise.py derives the tolerance); estimate_noise bit for
bit against denoise_ref.noise_sigma.  A frame's reference depends only on its window's frames and pairs, so it is
computed once per distinct window content and reused by the launches that read the same content.

Per-launch judging cannot see the wiring, because each launch is judged on whatever it read, so the wiring is checked bit
for bit (by content digests) from the logs:
  * denoise_video: the forwards' rows are pairs k0 + j of their batch, then padded pairs (P, P); slot p of flow_fw and
    flow_bw holds the logged forward and backward flow of pair p, slot T - 1 is zero and no padded pair is stored; sigma
    is the median of the logged estimates of frames 0 .. min(T, B + 1) - 1; the one denoise launch read the clip, frames
    0 .. T - 1 with t_hi = T - 1.
  * VideoDenoiser: at each launch every frame t of its window [max(t_lo, t0 - R), min(t_hi, t0 + n - 1 + R)] sits in
    ring slot t mod S and every pair t of [window start, window end - 1] in the flow slots t mod S, as the eager run's
    logged flows of that pair; launches follow each other with no gap and no repeat, from frame 0; each launch's t_hi is
    the last frame loaded before it in stream order (frame t and pair t - 1 stored on a stream whose record the
    denoising stream waited on), the final one T - 1; the yielded frames are the launches' out rows in order.
  * Ring hazards (host-order bookkeeping, not timing): for every store that overwrites frame or pair t - S, every
    launch whose window holds t - S was enqueued before the store, and the store's stream waited, before it, on an event
    the denoising stream recorded after the last of those launches.
Then the chain is restated with the batching removed: denoise_ref.denoise over the whole clip with the per-pair flows
gathered from the logged forwards (real pairs only) must pass _check against the chain's output, and VideoDenoiser must
equal denoise_video bit for bit, sigma included.

Runs (MaskFlownet-S and the cascade with random weights, flow heads scaled by FLOW_HEAD_SCALE so that some round trips
pass in each direction, under deterministic algorithms; a smooth texture panning (2, 1) px per frame with Gaussian noise
growing from sigma 8 to 12 over the clip): hd, MaskFlownet-S at batch 8 on 11 frames of 1080x1920 (a full batch, then 2
real and 6 padded pairs), radius 2; kitti, the cascade at batch 3 on 15 frames of 375x1242 (through the resize to
384x1280), radius 2 and 3 (rings of 11 and 13 slots, so they wrap); short, 64x64 clips of 2 and 1 frames at radius 13,
longer than the video (P = 1 and P = 0).  Asserted coverage: every kind of launch judged, the ring wrapped (kitti), padded
pairs (hd), and the share of output pixels that differ from the input within (0.005, 1).

Controls: each per-launch control (the fw and bw rings exchanged, the fw ring shifted by one pair, radius - 1,
sigma x 2; on every launch of hd and kitti, on its frame with the most neighbours) must miss _check by MARGIN, its share
beyond 1 at least MARGIN x FLIPPED or its inexact share at least MARGIN x (1 - EXACT), and each wiring control must
disagree with the chain (on kitti): pairs shifted by one (wiring checks failed), the last window clamped at t_hi - 1
(restated frames that fail _check), sigma from all frames (its distance from the chain's sigma), the ring's waits on the
denoising stream dropped (hazard checks failed).  test_denoise_chain_wiring_on_host runs the same recorder and the
denoise_video checks on the CPU, with the oracles standing in for the kernels and hand-made per-pair flows, at B = 3 and
P = 7: the right assignment passes, every launch control and every wiring control fails.
"""
import hashlib
import itertools
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch
from scipy.ndimage import gaussian_filter

from maskflownet_b200 import network, ops, video
from maskflownet_b200.video import VideoDenoiser
from oracle import denoise_ref as R

from launchcheck.denoise import EXACT, FLIPPED, _case, _check, _mismatch
from launchcheck.inputs import _deterministic, _scaled_model

MARGIN = 10.0           # how far a control must miss the judge (module docstring)
KINDS = ("denoise", "noise")
LAUNCH_CONTROLS = ("fw and bw rings exchanged", "fw ring shifted by one pair", "radius - 1", "sigma x 2")
WIRING_CONTROLS = ("pairs shifted by one", "last window clamped at t_hi - 1", "sigma from all frames",
                   "waits on the denoising stream dropped")
CHANGED = (0.005, 1.0)  # the share of output pixels that differ from the input lies strictly inside


def _sync():
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        torch.cuda.synchronize()


def _host(t):
    """A host copy (never a view: the rings change under it)."""
    t = t.detach()
    return (t.cpu() if t.is_cuda else t.clone()).numpy()


def _digest(a):
    return hashlib.blake2b(np.ascontiguousarray(a).tobytes(), digest_size=16).digest()


def _median(s):
    """ops.median_noise's rule: the lower middle value."""
    s = np.sort(np.asarray(s))
    return float(s[(len(s) - 1) // 2])


def _window(t0, n, t_lo, t_hi, radius):
    return max(t_lo, t0 - radius), min(t_hi, t0 + n - 1 + radius)


def _stream_of(t):
    return torch.cuda.current_stream(t.device).cuda_stream if t.is_cuda else 0


def _excess(got, ref):
    """How far a result misses the judge: max(share beyond 1 / FLIPPED, inexact share / (1 - EXACT))."""
    far, exact, _ = _mismatch(got, ref)
    return max(far / FLIPPED, (1.0 - exact) / (1.0 - EXACT))


# ------------------------------------------------------------------------------------------------------------------
# the float64 reference, frame by frame, once per distinct window content
# ------------------------------------------------------------------------------------------------------------------
class Oracle:
    def __init__(self, pool):
        self.pool, self.cache = pool, {}

    def frames(self, fr, fw, bw, ts, kw):
        """denoise_ref.denoise of frames ts of the rings (fr, fw, bw), kw: radius, sigma, h, patch, alpha, beta, t_lo,
        t_hi.  Frame t reads the frames of its window and the pairs before the window's end, nothing else."""
        S = len(fr)

        def one(t):
            a, b = _window(t, 1, kw["t_lo"], kw["t_hi"], kw["radius"])
            key = (tuple(_digest(fr[u % S]) for u in range(a, b + 1)),
                   tuple(_digest(fw[u % S]) + _digest(bw[u % S]) for u in range(a, b)), t - a, b - a,
                   tuple(float(kw[k]) for k in ("radius", "sigma", "h", "patch", "alpha", "beta")))
            if key not in self.cache:
                self.cache[key] = R.denoise(fr, fw, bw, kw["radius"], kw["sigma"], kw["h"], kw["patch"], kw["alpha"],
                                            kw["beta"], t0=t, n=1, t_lo=kw["t_lo"], t_hi=kw["t_hi"])[0]
            return self.cache[key]
        return np.stack(list(self.pool.map(one, ts)))


# ------------------------------------------------------------------------------------------------------------------
# the recorder
# ------------------------------------------------------------------------------------------------------------------
class DenoiseRecorder:
    """Wraps the entry points the denoising chain calls (`impl` replaces the originals: the host test passes the
    oracles).  begin(clip) starts a chain on a host clip; self.log holds its launches, stores and events in host order
    (each with its sequence number), self.pairs the logged (fw, bw) of each real pair and self.padded those of the
    padded pairs; self.judged counts the launches judged per kind; self.ctl the launch controls' (name, excess)."""

    def __init__(self, monkeypatch, impl=None, controls=False, workers=None, events=True):
        self.orig = dict(denoise_frames=ops.denoise_frames, estimate_noise=ops.estimate_noise,
                         _pair_flows=network._pair_flows, _store=video._FrameRing._store)
        self.orig.update(impl or {})
        rec = self
        monkeypatch.setattr(ops, "denoise_frames", self.denoise_frames)
        monkeypatch.setattr(ops, "estimate_noise", self.estimate_noise)
        monkeypatch.setattr(network, "_pair_flows", self._pair_flows)
        monkeypatch.setattr(video._FrameRing, "_store", lambda den, ring, src, t0: rec._store(den, ring, src, t0))
        if events:
            monkeypatch.setattr(torch.cuda, "Event", self._event_class())
        self.controls = controls
        self.pool = ThreadPoolExecutor(workers or min(8, os.cpu_count() or 1))
        self.oracle = Oracle(self.pool)
        self.seq = itertools.count()
        self.judged = {k: 0 for k in KINDS}
        self.ctl = []
        self.lines = []
        self.clip = None

    def begin(self, clip):
        self.clip = clip
        self.digests = [_digest(f) for f in clip]
        self.where = {d: t for t, d in enumerate(self.digests)}
        assert len(self.where) == len(clip), "the clip's frames must differ"
        self.log = {k: [] for k in ("flows", "noise", "denoise", "store", "events")}
        self.pairs, self.padded = {}, []

    def _tick(self):
        return next(self.seq)

    def _event_class(rec):
        uids = {}

        class LoggedEvent(torch.cuda.Event):
            """torch.cuda.Event that logs its records and the waits on it, with the stream, in host order."""

            def _uid(self):
                if id(self) not in uids:
                    uids[id(self)] = (len(uids), self)        # the reference keeps id() from being reused
                return uids[id(self)][0]

            def record(self, stream=None):
                stream = torch.cuda.current_stream() if stream is None else stream
                super().record(stream)
                if rec.clip is not None:
                    rec.log["events"].append(("record", self._uid(), stream.cuda_stream, rec._tick()))

            def wait(self, stream=None):
                stream = torch.cuda.current_stream() if stream is None else stream
                super().wait(stream)
                if rec.clip is not None:
                    rec.log["events"].append(("wait", self._uid(), stream.cuda_stream, rec._tick()))
        return LoggedEvent

    # ---- the forwards -------------------------------------------------------------------------------------------
    def _pair_flows(self, net, img1, img2, resize, bidirectional):
        flows = self.orig["_pair_flows"](net, img1, img2, resize, bidirectional)
        if img1.is_cuda and torch.cuda.is_current_stream_capturing():
            return flows
        _sync()
        f, N = _host(flows), len(img1)
        assert bidirectional and len(f) == 2 * N
        rows = [(self.where.get(_digest(a)), self.where.get(_digest(b)))
                for a, b in zip(_host(img1.permute(0, 2, 3, 1)), _host(img2.permute(0, 2, 3, 1)))]
        for r, (i, j) in enumerate(rows):
            if i is not None and j == i + 1:
                assert i not in self.pairs, f"pair {i} computed twice"
                self.pairs[i] = (f[r], f[N + r])
            elif i is not None and i == j:
                self.padded.append((f[r], f[N + r]))
        self.log["flows"].append(dict(rows=rows, seq=self._tick()))
        return flows

    # ---- the noise estimate -------------------------------------------------------------------------------------
    def estimate_noise(self, frames):
        s = self.orig["estimate_noise"](frames)
        _sync()
        f = _host(frames)
        f4 = f if f.ndim == 4 else f[None]
        got = np.atleast_1d(_host(s))
        assert np.array_equal(got, R.noise_sigma(f4)), f"estimate_noise launch {self.judged['noise']}"
        self.judged["noise"] += 1
        self.lines.append(f"noise    frames {[self.where.get(_digest(x)) for x in f4]}  bit-identical")
        self.log["noise"].append(dict(frames=[self.where.get(_digest(x)) for x in f4], sigma=got, seq=self._tick()))
        return s

    # ---- the ring ------------------------------------------------------------------------------------------------
    def _store(self, den, ring, src, t0):
        self.orig["_store"](den, ring, src, t0)
        _sync()
        name = next(k for k in ("frames", "fw", "bw") if den._v["ring"][k].data_ptr() == ring.data_ptr())
        s = _host(src)
        idx = list(range(t0, t0 + len(s)))
        self.log["store"].append(dict(ring=name, idx=idx, slots=[t % den.ring_size for t in idx],
                                      digests=[_digest(x) for x in s], stream=_stream_of(ring), seq=self._tick()))

    # ---- the denoising --------------------------------------------------------------------------------------------
    def denoise_frames(self, frames, flow_fw, flow_bw, radius, sigma, h=ops.DENOISE_H, patch=ops.DENOISE_PATCH,
                       alpha=0.01, beta=0.5, t0=0, n=None, t_lo=0, t_hi=None, out=None):
        seq = self._tick()
        res = self.orig["denoise_frames"](frames, flow_fw, flow_bw, radius, sigma, h, patch, alpha, beta, t0=t0, n=n,
                                          t_lo=t_lo, t_hi=t_hi, out=out)
        _sync()
        fr, fw, bw, got = (_host(x) for x in (frames, flow_fw, flow_bw, res))
        S = len(fr)
        t_hi = t_lo + S - 1 if t_hi is None else t_hi
        n = t_hi - t0 + 1 if n is None else n
        kw = dict(radius=radius, sigma=sigma, h=h, patch=patch, alpha=alpha, beta=beta, t_lo=t_lo, t_hi=t_hi)
        a, b = _window(t0, n, t_lo, t_hi, radius)
        ts = range(t0, t0 + n)
        ref = self.oracle.frames(fr, fw, bw, ts, kw)
        far, exact, dmax = _mismatch(got, ref)
        self.lines.append(f"denoise  frames {t0}..{t0 + n - 1}  window {a}..{b}  t_hi {t_hi}  exact {exact:.6f}  "
                          f"beyond 1 {far:.2e}  max {dmax}")
        _check(got, ref, f"denoise_frames launch {self.judged['denoise']} (frames {t0}..{t0 + n - 1})", FLIPPED)
        self.judged["denoise"] += 1
        if self.controls:       # on the launch's frame with the most neighbours
            t = max(ts, key=lambda u: min(radius, u - t_lo) + min(radius, t_hi - u))
            ctl = self._controls(fr, fw, bw, got[t - t0], t, kw)
            self.lines.append(f"  controls on frame {t}: " + ", ".join(f"{c} {x:.3g}" for c, x in ctl))
        self.log["denoise"].append(dict(
            t0=t0, n=n, t_lo=t_lo, t_hi=t_hi, radius=radius, sigma=float(sigma), window=(a, b), got=got,
            frames=[_digest(x) for x in fr], fw=[_digest(x) for x in fw], bw=[_digest(x) for x in bw],
            stream=_stream_of(frames), seq=seq))
        return res

    def _controls(self, fr, fw, bw, got, t, kw):
        """The launch controls on frame t: each changed rule's reference and how far the launch misses it."""
        def ctl(name):
            f, g, k = fw, bw, dict(kw)
            if name == "fw and bw rings exchanged":
                f, g = bw, fw
            elif name == "fw ring shifted by one pair":
                f = np.roll(fw, -1, axis=0)                 # slot t % S holds pair t + 1
            elif name == "radius - 1":
                k["radius"] = kw["radius"] - 1
            elif name == "sigma x 2":
                k["sigma"] = 2.0 * kw["sigma"]
            ref = R.denoise(fr, f, g, k["radius"], k["sigma"], k["h"], k["patch"], k["alpha"], k["beta"], t0=t, n=1,
                            t_lo=k["t_lo"], t_hi=k["t_hi"])
            return name, _excess(got[None], ref)
        names = [c for c in LAUNCH_CONTROLS if c != "radius - 1" or kw["radius"] >= 1]
        out = list(self.pool.map(ctl, names))
        self.ctl += out
        return out


# ------------------------------------------------------------------------------------------------------------------
# the wiring, from the logs of one chain (wrong assignments as `variant`, for the controls)
# ------------------------------------------------------------------------------------------------------------------
ZERO_FLOW = {}


def _zero_digest(H, W):
    if (H, W) not in ZERO_FLOW:
        ZERO_FLOW[(H, W)] = _digest(np.zeros((H, W, 2), np.float32))
    return ZERO_FLOW[(H, W)]


def _pair_digest(pairs, p, shift=0):
    q = p + shift
    return (_digest(pairs[q][0]), _digest(pairs[q][1])) if q in pairs else None


def _eager_wiring(rec, T, B, sigma, variant=None):
    log, P = rec.log, T - 1
    H, W = rec.clip.shape[1:3]
    m = min(T, B + 1)
    nb = -(-P // B) if P > 0 else 0
    w = {"launches: ceil(P/B) forwards, one estimate, one denoise (none for one frame)":
         len(log["flows"]) == nb and len(log["noise"]) == 1 and len(log["denoise"]) == (1 if T > 1 else 0)}
    if not all(w.values()):
        return w
    for i, fl in enumerate(log["flows"]):
        k0 = i * B
        want = [(k0 + j, k0 + j + 1) if k0 + j < P else (P, P) for j in range(B)]
        w[f"forward {i}: rows are pairs {k0}.. of the batch, then padded pairs (P, P)"] = fl["rows"] == want
    w["the real pairs 0..P-1 each computed once"] = sorted(rec.pairs) == list(range(P))
    noise = log["noise"][0]
    w[f"sigma: one estimate of frames 0..{m - 1}"] = noise["frames"] == list(range(m))
    want_sigma = _median(R.noise_sigma(rec.clip)) if variant == "sigma from all frames" else _median(noise["sigma"])
    w["sigma is the median of the estimates"] = sigma == want_sigma
    if T == 1:
        return w
    d = log["denoise"][0]
    t_hi = T - 2 if variant == "last window clamped at t_hi - 1" else T - 1
    w["the launch: frames 0..T-1 of the clip, t_lo 0, t_hi T-1, and the chain's sigma"] = \
        d["frames"] == rec.digests and (d["t0"], d["n"], d["t_lo"], d["t_hi"]) == (0, T, 0, t_hi) and \
        d["sigma"] == float(np.float64(sigma))
    shift = 1 if variant == "pairs shifted by one" else 0
    for p in range(P):
        w[f"slot {p}: pair {p}'s forward and backward flow"] = (d["fw"][p], d["bw"][p]) == _pair_digest(rec.pairs, p,
                                                                                                        shift)
    z = _zero_digest(H, W)
    w["slot T-1 of both flows is zero"] = d["fw"][P] == z and d["bw"][P] == z
    pad = {_digest(f) for fb in rec.padded for f in fb}
    w["no padded pair stored"] = not pad & (set(d["fw"]) | set(d["bw"]))
    return w


def _ordered_before(log, d, drop_waits=False):
    """Per stream, the host sequence number before which everything enqueued on it precedes launch d on the GPU: d's
    own stream up to d, and for each wait on d's stream before d, the stream and time of the record it waited on."""
    recs, bound = {}, {d["stream"]: d["seq"]}
    for kind, uid, stream, seq in log["events"]:
        if seq > d["seq"]:
            break
        if kind == "record":
            recs[uid] = (seq, stream)
        elif stream == d["stream"] and uid in recs and not drop_waits:
            rs, rstream = recs[uid]
            bound[rstream] = max(bound.get(rstream, -1), rs)
    return bound


def _stored(log, bound, ring):
    return {t for st in log["store"] if st["ring"] == ring and st["seq"] < bound.get(st["stream"], -1)
            for t in st["idx"]}


def _stream_wiring(rec, T, S, R_, eager_pairs, outs, variant=None):
    log, P = rec.log, T - 1
    L = log["denoise"]
    w = {"the frames yielded: T": len(outs) == T}
    if T == 1:
        w["one frame: no launch, the frame itself"] = not L and _digest(outs[0]) == rec.digests[0]
        return w
    w["launches: at least one, the first from frame 0"] = bool(L) and L[0]["t0"] == 0
    if not all(w.values()):
        return w
    shift = 1 if variant == "pairs shifted by one" else 0
    digests = {p: _pair_digest(eager_pairs, p) for p in range(P)}
    for st in log["store"]:
        for t, dg in zip(st["idx"], st["digests"]):
            if st["ring"] == "frames":
                ok = dg == rec.digests[min(t, P)]                 # padding repeats the last frame
            else:
                ok = t >= P or dg == digests[t][0 if st["ring"] == "fw" else 1]
            w[f"store of {st['ring']} {t}: its frame or pair"] = w.get(f"store of {st['ring']} {t}: its frame or pair",
                                                                        True) and ok
    for k, d in enumerate(L):
        a, b = d["window"]
        w[f"launch {k}: frames {a}..{b} in slots t mod S"] = all(d["frames"][t % S] == rec.digests[t]
                                                                  for t in range(a, b + 1))
        w[f"launch {k}: pairs {a}..{b - 1} in the flow slots t mod S"] = all(
            (d["fw"][t % S], d["bw"][t % S]) == _pair_digest(eager_pairs, t, shift) for t in range(a, b))
        if k:
            w[f"launch {k} starts where launch {k - 1} ended"] = d["t0"] == L[k - 1]["t0"] + L[k - 1]["n"]
        bound = _ordered_before(log, d)
        fr, fw, bw = (_stored(log, bound, r) for r in ("frames", "fw", "bw"))
        loaded = -1
        while loaded + 1 <= P and loaded + 1 in fr and (loaded + 1 == 0 or {loaded} <= fw & bw):
            loaded += 1
        last = loaded - 1 if variant == "last window clamped at t_hi - 1" and k == len(L) - 1 else loaded
        w[f"launch {k}: t_hi {d['t_hi']} is the last frame loaded before it ({loaded}), t_lo 0, radius and sigma"] = \
            d["t_hi"] == last and d["t_lo"] == 0 and d["radius"] == R_ and d["sigma"] == L[0]["sigma"]
    w["the final launch ends at T-1 with t_hi T-1"] = L[-1]["t0"] + L[-1]["n"] == T and L[-1]["t_hi"] == T - 1
    rows = [r for d in L for r in d["got"]]
    w["the yielded frames are the launches' out rows, in order"] = len(rows) == T and all(
        np.array_equal(x, y) for x, y in zip(rows, outs))
    return w


def _hazards(log, S, drop_waits=False):
    """For every store that overwrites frame or pair t - S: every launch that reads it was enqueued before the store,
    and the store's stream waited, before the store, on a record of the launches' stream after the last of them."""
    L, w = log["denoise"], {}
    for st in log["store"]:
        for t in st["idx"]:
            old = t - S
            if old < 0:
                continue
            span = (lambda d: d["window"]) if st["ring"] == "frames" else (lambda d: (d["window"][0], d["window"][1] - 1))
            readers = [d for d in L if span(d)[0] <= old <= span(d)[1]]
            key = f"{st['ring']} {t} over {old}"
            w[f"{key}: every launch reading {old} enqueued before (none after reaches back)"] = \
                all(d["seq"] < st["seq"] for d in readers)
            if readers:
                last = max(readers, key=lambda d: d["seq"])
                fake = dict(stream=st["stream"], seq=st["seq"])
                bound = _ordered_before(log, fake, drop_waits)
                w[f"{key}: the store waited on a record after launch frames {last['t0']}.."] = \
                    bound.get(last["stream"], -1) > last["seq"]
    return w


def _restate(rec, pairs, T, kw, ts=None):
    """denoise_ref.denoise over the whole clip, flows gathered from the logged forwards (real pairs; slot T-1 zero)."""
    H, W = rec.clip.shape[1:3]
    fw = np.zeros((T, H, W, 2), np.float32)
    bw = np.zeros_like(fw)
    for p, (f, b) in pairs.items():
        fw[p], bw[p] = f, b
    return rec.oracle.frames(rec.clip, fw, bw, range(T) if ts is None else ts, kw)


def _changed(clip, out):
    return float((np.asarray(out) != clip).any(-1).mean())


# ------------------------------------------------------------------------------------------------------------------
# one chain through the recorder: denoise_video, then VideoDenoiser on the same clip
# ------------------------------------------------------------------------------------------------------------------
def _run(rec, model, clip, B, radius, stream=True):
    T, P = len(clip), len(clip) - 1
    rec.begin(clip)
    dev = torch.device("cuda") if stream else torch.device("cpu")
    out, sigma = network.denoise_video(model, torch.from_numpy(clip).to(dev), batch=B, radius=radius)
    out = _host(out)
    eager = dict(log=rec.log, pairs=rec.pairs, padded=rec.padded, wiring=_eager_wiring(rec, T, B, sigma))
    kw = dict(radius=radius, sigma=sigma, h=ops.DENOISE_H, patch=ops.DENOISE_PATCH, alpha=0.01, beta=0.5, t_lo=0,
              t_hi=T - 1)
    far = {}
    if T > 1:
        _check(out, _restate(rec, rec.pairs, T, kw), "denoise_video restated without the batching", FLIPPED)
        far["pairs shifted by one"] = sum(not ok for ok in _eager_wiring(rec, T, B, sigma, "pairs shifted by one").values())
        if T >= 3:        # the last window clamped at t_hi - 1: the frames whose forward window reaches T - 1
            ts = range(max(0, T - 1 - radius), T - 1)
            ref = _restate(rec, rec.pairs, T, dict(kw, t_hi=T - 2), ts)
            far["last window clamped at t_hi - 1"] = sum(_excess(out[t:t + 1], ref[i:i + 1]) > 1.0
                                                         for i, t in enumerate(ts))
        far["sigma from all frames"] = abs(_median(R.noise_sigma(clip)) - sigma)
    res = dict(T=T, out=out, sigma=sigma, eager=eager, wiring_far=far, changed=_changed(clip, out))
    if not stream:
        return res
    den = VideoDenoiser(model, batch=B, radius=radius)
    rec.begin(clip)
    outs = list(den.run(iter(clip)))
    S = den.ring_size
    res.update(S=S, stream_log=rec.log, stream=_stream_wiring(rec, T, S, radius, eager["pairs"], outs),
               hazards=_hazards(rec.log, S),
               wrapped=any(t >= S for st in rec.log["store"] for t in st["idx"]))
    assert den.sigma_used == sigma, (den.sigma_used, sigma)
    for t, fr in enumerate(outs):
        assert np.array_equal(fr, out[t]), f"VideoDenoiser frame {t} differs from denoise_video"
    if T > 1:
        far["pairs shifted by one"] += sum(not ok for ok in _stream_wiring(rec, T, S, radius, eager["pairs"], outs,
                                                                           "pairs shifted by one").values())
        far["last window clamped at t_hi - 1 (stream wiring)"] = sum(
            not ok for ok in _stream_wiring(rec, T, S, radius, eager["pairs"], outs,
                                            "last window clamped at t_hi - 1").values())
        far["waits on the denoising stream dropped"] = sum(not ok for ok in _hazards(rec.log, S, True).values())
    return res


def _failed(w):
    return [k for k, ok in w.items() if not ok]


# ------------------------------------------------------------------------------------------------------------------
# CPU: the recorder and the denoise_video checks with the oracles standing in for the kernels
# ------------------------------------------------------------------------------------------------------------------
HB, HP, HH, HW = 3, 7, 24, 32          # batch, pairs, frame size of the host test


def _hand_flows(i, j, H, W):
    """The forward and backward flow a fake forward gives for frames (i, j): _case's flows (most chains run, some stop,
    NaN and inf spots, targets outside), drawn per pair, padded pairs (P, P) included."""
    _, fw, bw = _case(np.random.default_rng(1000 * i + j), 1, H, W)
    return fw[0], bw[0]


def _host_impl(clip):
    where = {_digest(f): t for t, f in enumerate(clip)}
    Tt = torch.from_numpy

    def _pair_flows(net, img1, img2, resize, bidirectional):
        H, W = img1.shape[2:]
        ids = [(where[_digest(a)], where[_digest(b)]) for a, b in zip(img1.permute(0, 2, 3, 1).numpy(),
                                                                       img2.permute(0, 2, 3, 1).numpy())]
        fl = [_hand_flows(i, j, H, W) for i, j in ids]
        return Tt(np.stack([f for f, _ in fl] + [b for _, b in fl]))

    def denoise_frames(frames, flow_fw, flow_bw, radius, sigma, h=ops.DENOISE_H, patch=ops.DENOISE_PATCH, alpha=0.01,
                       beta=0.5, t0=0, n=None, t_lo=0, t_hi=None, out=None):
        return Tt(R.denoise(frames.numpy(), flow_fw.numpy(), flow_bw.numpy(), radius, sigma, h, patch, alpha, beta,
                            t0=t0, n=n, t_lo=t_lo, t_hi=t_hi))

    def estimate_noise(frames):
        return Tt(R.noise_sigma(frames.numpy()))

    return dict(_pair_flows=_pair_flows, denoise_frames=denoise_frames, estimate_noise=estimate_noise)


def _pan_clip(seed, T, H, W, sigma=(8.0, 12.0)):
    """T uint8 frames (T,H,W,3): a smooth texture panning (2, 1) px per frame, with Gaussian noise whose sigma grows
    linearly from sigma[0] at frame 0 to sigma[1] at the last, so that the median estimate of the first frames differs
    from that of all of them."""
    rng = np.random.default_rng(seed)
    c = gaussian_filter(rng.random((H + T + 8, W + 2 * T + 8, 3), np.float32), (2, 2, 0))
    c = (c - c.min()) / (c.max() - c.min()) * 235 + 10
    out = np.empty((T, H, W, 3), np.uint8)
    for t in range(T):
        s = sigma[0] + (sigma[1] - sigma[0]) * t / max(T - 1, 1)
        y, x = 4 + T - t, 4 + 2 * (T - t)
        out[t] = np.clip(np.rint(c[y:y + H, x:x + W] + rng.normal(0, s, (H, W, 3))), 0, 255)
    return out


def test_denoise_chain_wiring_on_host(monkeypatch):
    """B = 3, P = 7 (pairs 3 + 3 + 1): network.denoise_video on the host with the oracles as its kernels; the wiring
    checks and the batch-free restatement pass, launch counts are the chain's, every launch control misses the judge by
    MARGIN and every wiring control disagrees with the chain."""
    clip = _pan_clip(5, HP + 1, HH, HW)
    rec = DenoiseRecorder(monkeypatch, impl=_host_impl(clip), controls=True, workers=1, events=False)
    r = _run(rec, None, clip, HB, 2, stream=False)
    monkeypatch.undo()
    w = r["eager"]["wiring"]
    assert w and all(w.values()), _failed(w)
    assert rec.judged == dict(denoise=1, noise=1), rec.judged
    assert len(r["eager"]["padded"]) == 2 and CHANGED[0] < r["changed"] < CHANGED[1], r["changed"]
    print("launch controls (excess over the judge):", rec.ctl)
    assert {c for c, _ in rec.ctl} == set(LAUNCH_CONTROLS) and all(x >= MARGIN for _, x in rec.ctl), rec.ctl
    print("wiring controls (checks / frames / grey levels):", r["wiring_far"])
    assert set(r["wiring_far"]) == set(WIRING_CONTROLS[:3]) and all(v > 0 for v in r["wiring_far"].values())
    # one frame: one estimate, no forward, no launch
    rec = DenoiseRecorder(monkeypatch, impl=_host_impl(clip[:1]), workers=1, events=False)
    r = _run(rec, None, clip[:1], HB, 2, stream=False)
    monkeypatch.undo()
    assert all(r["eager"]["wiring"].values()) and rec.judged == dict(denoise=0, noise=1)
    assert np.array_equal(r["out"], clip[:1])


# ------------------------------------------------------------------------------------------------------------------
# GPU: the runs
# ------------------------------------------------------------------------------------------------------------------
RUNS = {   # run: (model class, batch, [(frames, radius)], H, W, clip seed)
    "hd": (network.MaskFlownetS, 8, [(11, 2)], 1080, 1920, 101),
    "kitti": (network.MaskFlownet, 3, [(15, 2), (15, 3)], 375, 1242, 102),
    "short": (network.MaskFlownetS, 8, [(2, 13), (1, 13)], 64, 64, 103),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
def test_every_launch_of_the_denoising_chain_against_float64(run, monkeypatch):
    cls, B, cases, H, W, seed = RUNS[run]
    controls = run in ("hd", "kitti")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t_start = time.perf_counter()
    model = _scaled_model(cls)
    with _deterministic():
        rec = DenoiseRecorder(monkeypatch, controls=controls)
        results = []
        for T, radius in cases:
            results.append(_run(rec, model, _pan_clip(seed + T, T, H, W), B, radius))
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t_start, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    rec.pool.shutdown()

    for line in rec.lines:
        print(f"{run}: {line}")
    want = dict(denoise=0, noise=0)
    for r, (T, radius) in zip(results, cases):
        want["noise"] += 2
        want["denoise"] += (T > 1) * (1 + len(r["stream_log"]["denoise"]))
        print(f"{run} T={T} R={radius}: sigma {r['sigma']:.4f}, ring {r['S']} slots, wrapped {r['wrapped']}, padded "
              f"pairs {len(r['eager']['padded'])}, changed pixels {r['changed']:.4f}, stream launches "
              f"{[(d['t0'], d['t0'] + d['n'] - 1, d['window'], d['t_hi']) for d in r['stream_log']['denoise']]}")
        for name in ("stream", "hazards"):
            print(f"{run} T={T} R={radius} {name}: {len(r[name])} checks, failed {_failed(r[name])}")
        print(f"{run} T={T} R={radius} eager: {len(r['eager']['wiring'])} checks, failed "
              f"{_failed(r['eager']['wiring'])}")
    print(f"{run}: launches judged {rec.judged}; {secs:.1f} s, peak {peak:.2f} GiB allocated")

    assert rec.judged == want and all(rec.judged.values()), (rec.judged, want)
    for r in results:
        for w in (r["eager"]["wiring"], r["stream"]):
            assert w and all(w.values()), _failed(w)
        assert all(r["hazards"].values()), _failed(r["hazards"])       # empty where the ring never wraps
    if run == "hd":
        assert len(results[0]["eager"]["padded"]) == 6
    if run == "kitti":
        assert all(r["wrapped"] for r in results)
    if run in ("hd", "kitti"):
        for r in results:
            assert CHANGED[0] < r["changed"] < CHANGED[1], r["changed"]
    if controls:
        for name in LAUNCH_CONTROLS:
            x = [e for c, e in rec.ctl if c == name]
            print(f"{run} launch control {name}: {len(x)} launches, excess over the judge min {min(x):.3g} max "
                  f"{max(x):.3g} (must be >= {MARGIN:g})")
            assert x and min(x) >= MARGIN, (name, x)
    if run == "kitti":         # the wrapped ring gives the dropped waits something to break
        for r, (T, radius) in zip(results, cases):
            print(f"kitti R={radius} wiring controls (checks / frames / grey levels):", r["wiring_far"])
            assert set(WIRING_CONTROLS) <= set(r["wiring_far"]) and all(v > 0 for v in r["wiring_far"].values()), \
                r["wiring_far"]
