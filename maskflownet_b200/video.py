"""Streaming flow over a video: consecutive frame pairs in, Middlebury colour images (and optionally the flows) out.

What predict_new_data.py does with a video -- pipe.predict over (frame t, frame t+1) pairs, then flow_vis.flow_to_color
on the host -- as one CUDA graph per frame size, with every frame crossing PCIe once and only uint8 colours coming back.

A batch of B pairs reads B+1 consecutive frames.  They sit in one static device buffer F (B+1, H, W, 3): the pairs' first
images are F[:B] and their second images F[1:], both contiguous views.  Between batches F[0] <- F[B] on the compute stream
and the next B frames go into F[1:].  The graph holds the whole chain:
    HWC -> NCHW  ->  ops.preprocess (/255, centralise, resize to padded_size)  ->  network  ->  ops.postprocess
    (Upsample(4), resize back, (x,y) NHWC)  ->  ops.flow_to_color
With bidirectional=True the network's bidirectional forward (one feature pyramid for both directions of each pair) gives
2B flows, postprocess takes them all, the forward flows are coloured and ops.flow_consistency gives both occlusion masks:
    preprocess(F[:B], F[1:])  ->  bidirectional forward  ->  postprocess (2B flows)  ->  flow_to_color (forward flows)
    ->  flow_consistency
With interpolate=T the chain continues into ops.interpolate_frames, which reads the frame buffer's two views directly, and
the colour coding is skipped:
    preprocess(F[:B], F[1:])  ->  bidirectional forward  ->  postprocess (2B flows)  ->  flow_consistency
    ->  interpolate_frames(F[:B], F[1:], ...) at the times k / (T+1), k = 1..T
VideoTracker extends the bidirectional chain with dense point tracking (ops.track_*) and yields one TrackFrame per
video frame:
    preprocess(F[:B], F[1:])  ->  bidirectional forward  ->  postprocess (2B flows)  ->  track_texture(F)
    ->  per pair: track_advance, track_seed
VideoStabilizer extends the one-direction chain with the camera's motion per pair (ops.affine_motion); the camera path is
smoothed on the host (camera.stabilize_path) and the frames, kept on the device in a ring, are warped outside the graph:
    preprocess(F[:B], F[1:])  ->  network  ->  postprocess  ->  affine_motion
VideoMotionSegmenter extends the bidirectional chain with the camera-relative motion of both directions and the objects
it forms (ops.segment_motion), carrying the last backward residual of each batch into the next on the device:
    preprocess(F[:B], F[1:])  ->  bidirectional forward  ->  postprocess (2B flows)  ->  flow_consistency
    ->  affine_motion (2B flows, residuals)  ->  segment_motion (B frames)
VideoDenoiser ends the bidirectional chain at the 2B flows; each batch's frames and flows are copied into a device ring,
and the frames whose window of neighbours is complete are denoised outside the graph (ops.denoise_frames):
    preprocess(F[:B], F[1:])  ->  bidirectional forward  ->  postprocess (2B flows)
Copies follow network.PipelinedFlowPredictor's slot scheme: pinned host staging, H2D on one copy stream, D2H of the colours
(and flows) on another, `depth` slots, so the copies of neighbouring batches run under the replay of this one.
"""
from __future__ import annotations

import collections
import itertools
from typing import Iterable, Iterator, NamedTuple

import numpy as np
import torch
import torch.nn as nn

from . import camera, network, ops
from ._lib import MaskflowError

_WARMUP = 2


class _FrameRing:
    """The bookkeeping of a device ring of `ring_size` slots that holds frame t in slot t % ring_size (VideoStabilizer's
    frames waiting for their warp, VideoDenoiser's frames and flows waiting for their window)."""
    ring_size: int

    def _segments(self, t0: int, t1: int):
        """Frames [t0, t1) as runs that are contiguous in the ring."""
        n, out = self.ring_size, []
        while t0 < t1:
            b = min(t1, t0 + n - t0 % n)
            out.append((t0, b))
            t0 = b
        return out

    def _store(self, ring: torch.Tensor, src: torch.Tensor, t0: int) -> None:
        """Copies frames t0 .. t0 + len(src) - 1 (src[0] is frame t0) into their slots of `ring`."""
        n = self.ring_size
        for a, b in self._segments(t0, t0 + len(src)):
            ring[a % n:a % n + (b - a)].copy_(src[a - t0:b - t0])


class VideoFlowPredictor:
    """run(frames) yields one result per consecutive pair (t, t+1), in order: the colour image (H,W,3) uint8, or
    (colour, flow (H,W,2) float32 (x,y) pixels) with want_flow -- the layouts of PipelineFlownet.predict.

    frames: host uint8 (H,W,3) arrays or tensors, in the channel order given (no BGR/RGB swap, like the reference feeding
    cv2 frames to pipe.predict); every frame must have the first one's size.  batch: pairs per graph replay; the last,
    partial batch repeats the last frame in its unused slots and yields only its real pairs.  resize: the network input
    size (H', W'), default the next multiples of 64.  max_radius / bgr: as ops.flow_to_color; a fixed max_radius keeps the
    colours of successive frames comparable.

    bidirectional: each pair is also predicted backwards, (t+1 -> t), from the same feature pyramid, and each result
    appends the forward-backward occlusion masks (H,W) uint8 (ops.flow_consistency with alpha, beta): occ_fw marks the
    pixels of frame t with no consistent match in frame t+1, occ_bw those of frame t+1 with none in frame t.  Results are
    (colour, occ_fw, occ_bw), or with want_flow (colour, flow, flow_bw, occ_fw, occ_bw); the masks and the backward flow
    take the same slots and copy streams as the colours.

    interpolate: T >= 1 in-between frames per pair instead of the colour image, at the uniform times k / (T+1), k = 1..T
    (ops.interpolate_frames, occluded pixels weighted by occ_weight); implies bidirectional.  Results are the (T,H,W,3)
    uint8 stack of pair (t, t+1), in the channel order of the frames, or with want_flow (frames, flow, flow_bw, occ_fw,
    occ_bw).  interpolate=0 (default): no interpolation.

    Weights are read through the packed images cached in the model: call invalidate() after changing parameters.  Graphs are kept per frame size and network.precision_key of the model."""

    def __init__(self, net: nn.Module, batch: int = 8, resize=None, max_radius=None, bgr: bool = False,
                 want_flow: bool = False, depth: int = 2, bidirectional: bool = False, alpha: float = 0.01,
                 beta: float = 0.5, interpolate: int = 0, occ_weight: float = 0.01):
        if batch < 1 or depth < 1:
            raise MaskflowError(f"VideoFlowPredictor: batch and depth must be >= 1 (got {batch}, {depth})")
        if max_radius is not None and not (0.0 < float(max_radius) < float("inf")):
            raise MaskflowError(f"VideoFlowPredictor: max_radius must be positive and finite, got {max_radius}")
        self.net, self.batch, self.depth = net, int(batch), int(depth)
        self.resize = None if resize is None else (int(resize[0]), int(resize[1]))
        self.max_radius, self.bgr, self.want_flow = max_radius, bool(bgr), bool(want_flow)
        if not isinstance(interpolate, int) or isinstance(interpolate, bool) or interpolate < 0:
            raise MaskflowError(f"VideoFlowPredictor: interpolate must be a non-negative integer, got {interpolate!r}")
        if interpolate and not 0.0 <= float(occ_weight) <= 1.0:
            raise MaskflowError(f"VideoFlowPredictor: occ_weight must lie in [0,1], got {occ_weight}")
        bidirectional = bool(bidirectional) or interpolate > 0
        if bidirectional and not (0.0 <= float(alpha) < float("inf") and 0.0 <= float(beta) < float("inf")):
            raise MaskflowError(f"VideoFlowPredictor: alpha and beta must be finite and non-negative, got {alpha}, {beta}")
        self.bidirectional, self.alpha, self.beta = bidirectional, float(alpha), float(beta)
        self.interpolate, self.occ_weight = int(interpolate), float(occ_weight)
        self._states = {}
        self._streams = None

    def invalidate(self) -> None:
        self._states.clear()

    # ---- one graph per frame size ------------------------------------------------------------------------------
    def _chain(self, F: torch.Tensor, H: int, W: int):
        """The captured chain: {"rgb", "flow"}, and with bidirectional also {"flow_bw", "occ_fw", "occ_bw"}; with
        interpolate {"frames", "flow", "flow_bw", "occ_fw", "occ_bw"}."""
        B = self.batch
        flows = network._frame_pair_flows(self.net, F, self.resize, self.bidirectional)
        if not self.bidirectional:
            rgb, _ = ops.flow_to_color(flows, self.max_radius, self.bgr)
            return {"rgb": rgb, "flow": flows}
        flow, flow_bw = flows[:B], flows[B:]
        if self.interpolate:
            occ_fw, occ_bw = ops.flow_consistency(flow, flow_bw, self.alpha, self.beta)
            times = [k / (self.interpolate + 1) for k in range(1, self.interpolate + 1)]
            frames = ops.interpolate_frames(F[:B], F[1:], flow, flow_bw, occ_fw, occ_bw, times, self.occ_weight)
            return {"frames": frames, "flow": flow, "flow_bw": flow_bw, "occ_fw": occ_fw, "occ_bw": occ_bw}
        rgb, _ = ops.flow_to_color(flow, self.max_radius, self.bgr)
        occ_fw, occ_bw = ops.flow_consistency(flow, flow_bw, self.alpha, self.beta)
        return {"rgb": rgb, "flow": flow, "flow_bw": flow_bw, "occ_fw": occ_fw, "occ_bw": occ_bw}

    def _outputs(self):
        """The chain outputs that leave the GPU, in the order of a result."""
        if self.interpolate:
            return ("frames", "flow", "flow_bw", "occ_fw", "occ_bw") if self.want_flow else ("frames",)
        if not self.bidirectional:
            return ("rgb", "flow") if self.want_flow else ("rgb",)
        return ("rgb", "flow", "flow_bw", "occ_fw", "occ_bw") if self.want_flow else ("rgb", "occ_fw", "occ_bw")

    def _state(self, H: int, W: int, dev: torch.device):
        key = (H, W, network.precision_key(self.net))
        st = self._states.get(key)
        if st is not None:
            return st
        B = self.batch
        F = torch.zeros((B + 1, H, W, 3), dtype=torch.uint8, device=dev)
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):      # warm-up off the capture: weight packing, kernel attributes
            for _ in range(_WARMUP):
                self._chain(F, H, W)
        cur.wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = self._chain(F, H, W)
        slots = []
        for _ in range(self.depth):
            s = {"in": torch.empty((B + 1, H, W, 3), dtype=torch.uint8, device=dev),
                 "in_host": torch.empty((B + 1, H, W, 3), dtype=torch.uint8, pin_memory=True),
                 "ev_h2d": torch.cuda.Event(), "ev_in_free": torch.cuda.Event(), "ev_out": torch.cuda.Event(),
                 "ev_out_free": torch.cuda.Event(), "used": False}
            for name in self._outputs():
                s[name] = torch.empty_like(out[name])
                s[name + "_host"] = torch.empty(out[name].shape, dtype=out[name].dtype, pin_memory=True)
            slots.append(s)
        st = self._states[key] = {"graph": graph, "F": F, "out": out, "slots": slots, "i": 0}
        return st

    # ---- one batch ---------------------------------------------------------------------------------------------
    def _submit(self, st, frames, first: bool):
        """Enqueue one batch: frames are B+1 host frames for the first batch of a video, B afterwards."""
        B = self.batch
        s = st["slots"][st["i"] % self.depth]
        st["i"] += 1
        dev = st["F"].device
        h2d, d2h = self._streams
        cur = torch.cuda.current_stream(dev)
        if s["used"]:
            s["ev_h2d"].synchronize()               # the pinned staging of this slot's previous batch has been read
        for j, fr in enumerate(frames):
            s["in_host"][j].copy_(fr)
        k = len(frames)
        with torch.cuda.stream(h2d):
            if s["used"]:
                h2d.wait_event(s["ev_in_free"])
            s["in"][:k].copy_(s["in_host"][:k], non_blocking=True)
            s["ev_h2d"].record(h2d)
        cur.wait_event(s["ev_h2d"])
        F = st["F"]
        if first:
            F.copy_(s["in"])
            self._start(st)
        else:
            F[0].copy_(F[B])
            F[1:].copy_(s["in"][:B])
        self._loaded(st, first)
        s["ev_in_free"].record(cur)
        st["graph"].replay()
        self._replayed(st)
        if s["used"]:
            cur.wait_event(s["ev_out_free"])
        for name in self._outputs():
            s[name].copy_(st["out"][name])
        s["ev_out"].record(cur)
        with torch.cuda.stream(d2h):
            d2h.wait_event(s["ev_out"])
            for name in self._outputs():
                s[name + "_host"].copy_(s[name], non_blocking=True)
            s["ev_out_free"].record(d2h)
        s["used"] = True
        return s

    def _start(self, st) -> None:
        """Runs on the compute stream once per video, after frame 0 is in the frame buffer and before the first replay."""

    def _loaded(self, st, first: bool) -> None:
        """Runs on the compute stream once per batch, after the batch's new frames are in the frame buffer (F[0..B] for
        the first batch of a video, F[1..B] afterwards) and before its replay."""

    def _replayed(self, st) -> None:
        """Runs on the compute stream once per batch, right after its replay, while the graph's outputs hold it."""

    def _collect(self, s, b: int) -> Iterator:
        s["ev_out_free"].synchronize()
        names = self._outputs()
        for j in range(b):
            res = tuple(s[name + "_host"][j].numpy().copy() for name in names)
            yield res if len(res) > 1 else res[0]

    @staticmethod
    def _frame(fr, hw) -> torch.Tensor:
        t = torch.as_tensor(np.ascontiguousarray(fr) if isinstance(fr, np.ndarray) else fr)
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
            raise MaskflowError(f"VideoFlowPredictor: frames must be uint8 (H,W,3), got {t.dtype} {tuple(t.shape)}")
        if hw is not None and tuple(t.shape[:2]) != hw:
            raise MaskflowError(f"VideoFlowPredictor: frame of size {tuple(t.shape[:2])} in a video of size {hw}")
        return t

    @torch.no_grad()
    def run(self, frames: Iterable) -> Iterator:
        it = iter(frames)
        first = next(it, None)
        if first is None:
            return
        first = self._frame(first, None)
        H, W = int(first.shape[0]), int(first.shape[1])
        dev = next(self.net.parameters()).device
        B = self.batch
        with torch.cuda.device(dev):
            st = self._state(H, W, dev)
            if self._streams is None:
                self._streams = (torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev))
        pending = collections.deque()
        buf, first_batch = [first], True      # the first batch also uploads frame 0
        for fr in it:
            buf.append(self._frame(fr, (H, W)))
            if len(buf) == (B + 1 if first_batch else B):
                with torch.cuda.device(dev):
                    pending.append((self._submit(st, buf, first_batch), B))
                buf, first_batch = [], False
                if len(pending) >= self.depth:
                    yield from self._collect(*pending.popleft())
        pairs = len(buf) - (1 if first_batch else 0)
        if pairs > 0:
            buf += [buf[-1]] * ((B + 1 if first_batch else B) - len(buf))
            with torch.cuda.device(dev):
                pending.append((self._submit(st, buf, first_batch), pairs))
        while pending:
            yield from self._collect(*pending.popleft())


# ---------------------------------------------------------------------------------------------------------------------
# Dense point tracking
# ---------------------------------------------------------------------------------------------------------------------
class TrackFrame(NamedTuple):
    """The tracks of one video frame.  ids (n,) int64, xy (n,2) float32 (x,y) pixels and born (n,) bool: the tracks alive
    in this frame (born: started in it); ended_ids (m,) int64 and ended_reason (m,) uint8 (ops.TRACK_LEFT,
    TRACK_OCCLUDED or TRACK_BOUNDARY): the tracks whose last frame was the previous one.  Query i has id i and is reported
    as ended with TRACK_LEFT in its frame if its point lies outside the frame; dense tracks count on from the number of
    queries, in order of birth frame, then slot."""
    ids: np.ndarray
    xy: np.ndarray
    born: np.ndarray
    ended_ids: np.ndarray
    ended_reason: np.ndarray


class _TrackIds:
    """Host bookkeeping: slot -> track id, from each frame's slot positions and status bytes."""

    def __init__(self, M: int):
        self.M, self.next, self.slot = M, M, None

    def frame(self, xy: np.ndarray, status: np.ndarray) -> TrackFrame:
        if self.slot is None:
            self.slot = np.full(len(status), -1, np.int64)
            self.slot[:self.M] = np.arange(self.M)
        born = status == ops.TRACK_BORN
        new = np.flatnonzero(born[self.M:]) + self.M
        self.slot[new] = np.arange(self.next, self.next + len(new))
        self.next += len(new)
        alive = born | (status == ops.TRACK_TRACKED)
        ended = status >= ops.TRACK_LEFT
        res = TrackFrame(self.slot[alive], xy[alive], born[alive], self.slot[ended], status[ended])
        ended[:self.M] = False
        self.slot[ended] = -1                 # a dense slot may be seeded again from the next frame on
        return res


def track_frames(xy, status, num_queries: int = 0) -> Iterator[TrackFrame]:
    """TrackFrames from per-frame slot arrays, xy (T,K,2) and status (T,K) (network.track_video's first two results,
    on the host), num_queries = M."""
    ids = _TrackIds(int(num_queries))
    for k in range(len(status)):
        yield ids.frame(np.asarray(xy[k]), np.asarray(status[k]))


def collect_tracks(frames: Iterable[TrackFrame]):
    """Ragged arrays of the tracks in a sequence of TrackFrames (frame 0 first), indexed by track id: "start" (n,) int64,
    the first frame (-1 for an id never seen); "length" (n,) int64, the frames it was alive in; "offset" (n,) int64 into
    "xy" (sum(length), 2) float32, its positions frame by frame; "reason" (n,) uint8, how it ended (0 = still alive in the
    last frame).  A query whose point lay outside its frame has length 0, its frame as start and reason TRACK_LEFT."""
    ids, ts, xys, eids, ets, ereasons = [], [], [], [], [], []
    for t, fr in enumerate(frames):
        ids.append(np.asarray(fr.ids, np.int64))
        ts.append(np.full(len(fr.ids), t, np.int64))
        xys.append(np.asarray(fr.xy, np.float32).reshape(-1, 2))
        eids.append(np.asarray(fr.ended_ids, np.int64))
        ets.append(np.full(len(fr.ended_ids), t, np.int64))
        ereasons.append(np.asarray(fr.ended_reason, np.uint8))
    cat = lambda a, dt: np.concatenate(a) if a else np.zeros(0, dt)   # noqa: E731
    ids, ts, eids, ets, ereasons = cat(ids, np.int64), cat(ts, np.int64), cat(eids, np.int64), cat(ets, np.int64), \
        cat(ereasons, np.uint8)
    xy = np.concatenate(xys) if xys else np.zeros((0, 2), np.float32)
    n = int(max(ids.max(initial=-1), eids.max(initial=-1))) + 1
    order = np.argsort(ids, kind="stable")
    length = np.bincount(ids, minlength=n).astype(np.int64)
    offset = np.cumsum(length) - length
    start = np.full(n, -1, np.int64)
    has = length > 0
    start[has] = ts[order][offset[has]]
    reason = np.zeros(n, np.uint8)
    reason[eids] = ereasons
    unborn = np.zeros(n, bool)
    unborn[eids] = True
    unborn &= ~has
    start[eids[unborn[eids]]] = ets[unborn[eids]]
    return {"start": start, "length": length, "offset": offset, "xy": xy[order], "reason": reason}


class VideoTracker(VideoFlowPredictor):
    """Dense point tracks through a video, streamed: run(frames) yields one TrackFrame per video frame, frame 0 included.

    The pairs go through VideoFlowPredictor's bidirectional machinery (frame buffer, pinned slots, copy streams, one CUDA
    graph per frame size and network.precision_key), and the graph continues after postprocess with the tracking steps
    of network.track_video: one ops.track_texture over the batch's B+1 frames, then per pair ops.track_advance and
    ops.track_seed.  The tracker's state (ops.TrackState: spacing, tau, alpha, beta, boundary, max_tracks, queries) lives
    on the device; run() resets it and seeds frame 0 before its first replay.  Only the slot positions and status bytes
    cross PCIe (9 bytes per slot and frame); track ids are assigned on the host.  The padded tail of a partial batch is
    discarded.  frames: host uint8 (H,W,3) arrays or tensors, any channel order.  collect_tracks turns the TrackFrames
    into ragged arrays."""

    def __init__(self, net: nn.Module, batch: int = 8, resize=None, spacing: int = 8, tau: float = 0.001,
                 alpha: float = 0.01, beta: float = 0.5, boundary=(0.01, 0.002), max_tracks=None, queries=None,
                 depth: int = 2):
        super().__init__(net, batch=batch, resize=resize, depth=depth, bidirectional=True, alpha=alpha, beta=beta)
        q = ops.check_track_args(spacing, None if queries is None else np.asarray(queries, np.float64), "VideoTracker")
        self.track_args = dict(spacing=spacing, tau=tau, alpha=alpha, beta=beta, boundary=boundary, max_tracks=max_tracks,
                               queries=None if queries is None else q.numpy())
        self.num_queries = int(q.shape[0])
        self._tracks = {}
        self._first = None

    def invalidate(self) -> None:
        super().invalidate()
        self._tracks.clear()

    def _track(self, H: int, W: int, dev: torch.device):
        """The device state of H x W videos and the buffers of frame 0's result."""
        e = self._tracks.get((H, W))
        if e is None:
            st = ops.TrackState(H, W, **self.track_args, device=dev)
            e = self._tracks[(H, W)] = {
                "state": st, "xy0": torch.empty((st.K, 2), dtype=torch.float32, device=dev),
                "status0": torch.empty((st.K,), dtype=torch.uint8, device=dev),
                "dropped0": torch.empty((1,), dtype=torch.int32, device=dev),
                "xy0_host": torch.empty((st.K, 2), dtype=torch.float32, pin_memory=True),
                "status0_host": torch.empty((st.K,), dtype=torch.uint8, pin_memory=True), "ev0": torch.cuda.Event()}
        return e

    def _chain(self, F: torch.Tensor, H: int, W: int):
        st = self._track(H, W, F.device)["state"]
        flows = network._frame_pair_flows(self.net, F, self.resize, True)
        xy, status, dropped = network._track_batch(st, F, flows, self.batch)
        return {"xy": xy, "status": status, "dropped": dropped}

    def _outputs(self):
        return ("xy", "status")

    def _start(self, st) -> None:
        F = st["F"]
        e = self._track(F.shape[1], F.shape[2], F.device)
        ops.track_start(e["state"], F[0], e["xy0"], e["status0"], e["dropped0"])
        e["xy0_host"].copy_(e["xy0"], non_blocking=True)
        e["status0_host"].copy_(e["status0"], non_blocking=True)
        e["ev0"].record()
        self._first = e

    def _collect(self, s, b: int) -> Iterator:
        if self._first is not None:
            e, self._first = self._first, None
            e["ev0"].synchronize()
            yield e["xy0_host"].numpy().copy(), e["status0_host"].numpy().copy()
        yield from super()._collect(s, b)

    @torch.no_grad()
    def run(self, frames: Iterable) -> Iterator[TrackFrame]:
        ids = _TrackIds(self.num_queries)
        it = iter(frames)
        head = [fr for fr in (next(it, None), next(it, None)) if fr is not None]
        if not head:
            return
        if len(head) == 1:                   # one frame: no pair, only its seeds
            fr = self._frame(head[0], None)
            dev = next(self.net.parameters()).device
            with torch.cuda.device(dev):
                e = self._track(int(fr.shape[0]), int(fr.shape[1]), dev)
                ops.track_start(e["state"], fr.to(dev).contiguous(), e["xy0"], e["status0"], e["dropped0"])
                yield ids.frame(e["xy0"].cpu().numpy(), e["status0"].cpu().numpy())
            return
        for xy, status in super().run(itertools.chain(head, it)):
            yield ids.frame(xy, status)


# ---------------------------------------------------------------------------------------------------------------------
# Video stabilisation
# ---------------------------------------------------------------------------------------------------------------------
class VideoStabilizer(_FrameRing, VideoFlowPredictor):
    """A stabilised video, streamed: run(frames) yields one stabilised (H,W,3) uint8 frame per input frame, frame 0
    included, in order, `radius` frames behind the input.

    The pairs go through VideoFlowPredictor's one-direction machinery (frame buffer, pinned slots, copy streams, one CUDA
    graph per frame size and network.precision_key), and the graph continues after postprocess with ops.affine_motion
    (iterations, sigma): only the fit of each pair, 6 doubles and an ok byte, comes back to the host.  There
    camera.stabilize_path turns the fits into one warp per frame (smoothing window `radius`, zoom `crop`; a pair whose fit
    failed counts as no motion) once the fits of the frame's window are in.  The frames wait for their warp on the device,
    in a ring of radius + depth * batch + 1 frames filled from the frame buffer on the compute stream; once per collected
    batch, ops.warp_frames_affine warps the frames that became ready, on a stream of its own.  Each frame crosses PCIe once
    in each direction, and host memory is bounded by the radius and the batch, not the video's length.  The results
    equal network.stabilize_video's bit for bit.  frames: host uint8 (H,W,3) arrays or tensors, any channel order."""

    def __init__(self, net: nn.Module, batch: int = 8, resize=None, radius: int = 15, crop: float = 0.9,
                 iterations: int = ops.AFFINE_ITERATIONS, sigma: float = ops.AFFINE_SIGMA,
                 depth: int = 2):
        super().__init__(net, batch=batch, resize=resize, depth=depth)
        camera.check_path_args(radius, crop, "VideoStabilizer")
        ops.check_affine_args(iterations, sigma, "VideoStabilizer")
        self.radius, self.crop, self.iterations, self.sigma = int(radius), float(crop), int(iterations), float(sigma)
        self.ring_size = self.radius + self.depth * self.batch + 1
        self._rings = {}
        self._v = None          # the state of the video being run

    def invalidate(self) -> None:
        super().invalidate()
        self._rings.clear()

    def _chain(self, F: torch.Tensor, H: int, W: int):
        flow = network._frame_pair_flows(self.net, F, self.resize, False)
        affine, ok = ops.affine_motion(flow, self.iterations, self.sigma)
        return {"affine": affine, "ok": ok}

    def _outputs(self):
        return ("affine", "ok")

    def _ring(self, H: int, W: int, dev: torch.device):
        """The device ring of frames waiting for their warp, its output buffers and the warp stream."""
        e = self._rings.get((H, W))
        if e is None:
            n = self.ring_size
            e = self._rings[(H, W)] = {
                "frames": torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev),
                "out": torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev),
                "out_host": torch.empty((n, H, W, 3), dtype=torch.uint8, pin_memory=True),
                "stream": torch.cuda.Stream(device=dev), "ev_ring": torch.cuda.Event(), "ev_warp": torch.cuda.Event(),
                "ev_host": torch.cuda.Event(), "warped": False}
        return e

    def _loaded(self, st, first: bool) -> None:
        """Copies the batch's new frames from the frame buffer into the ring, after the warps that read their slots."""
        F = st["F"]
        v = self._v
        r = v["ring"]
        cur = torch.cuda.current_stream(F.device)
        if r["warped"]:
            cur.wait_event(r["ev_warp"])
        src = F if first else F[1:]
        self._store(r["frames"], src, v["loaded"])
        v["loaded"] += len(src)
        r["ev_ring"].record(cur)

    def _warp_ready(self, n_frames=None) -> list:
        """Warps the frames whose smoothing window is known and returns them on the host: all the rest when n_frames (the
        video's length) is given, else those t with t + radius <= the last frame whose path is known."""
        v = self._v
        known = len(v["P"]) + v["P0"] - 1          # P_0 .. P_known are known
        t0 = v["next"]
        t1 = n_frames if n_frames is not None else known - self.radius + 1
        if t1 <= t0:
            return []
        n = known + 1 if n_frames is None else n_frames
        M = np.stack([camera.stabilize_path(v["P"], t, n, v["H"], v["W"], self.radius, self.crop, v["P0"])
                      for t in range(t0, t1)])
        r = v["ring"]
        ws = r["stream"]
        with torch.cuda.stream(ws):
            ws.wait_event(r["ev_ring"])
            Md = torch.from_numpy(M).to(v["dev"])
            for a, b in self._segments(t0, t1):
                i = a % self.ring_size
                r["out"][a - t0:b - t0].copy_(ops.warp_frames_affine(r["frames"][i:i + (b - a)], Md[a - t0:b - t0]))
            r["ev_warp"].record(ws)
            r["warped"] = True
            r["out_host"][:t1 - t0].copy_(r["out"][:t1 - t0], non_blocking=True)
            r["ev_host"].record(ws)
        r["ev_host"].synchronize()
        v["next"] = t1
        drop = min(max(0, t1 - self.radius - v["P0"]), len(v["P"]) - 1)   # P_s, s < next - radius, is no longer needed
        del v["P"][:drop]
        v["P0"] += drop
        return [r["out_host"][j].numpy().copy() for j in range(t1 - t0)]

    def _collect(self, s, b: int) -> Iterator:
        s["ev_out_free"].synchronize()
        v = self._v
        aff, ok = s["affine_host"], s["ok_host"]
        for j in range(b):
            v["P"].append(camera.path_step(v["P"][-1], aff[j].numpy(), bool(ok[j])))
        with torch.cuda.device(v["dev"]):
            ready = self._warp_ready()
        yield from ready

    @torch.no_grad()
    def run(self, frames: Iterable) -> Iterator[np.ndarray]:
        it = iter(frames)
        head = [fr for fr in (next(it, None), next(it, None)) if fr is not None]
        if not head:
            return
        fr0 = self._frame(head[0], None)
        H, W = int(fr0.shape[0]), int(fr0.shape[1])
        dev = next(self.net.parameters()).device
        with torch.cuda.device(dev):
            self._v = {"H": H, "W": W, "dev": dev, "ring": self._ring(H, W, dev), "loaded": 0, "next": 0,
                       "P": [np.eye(3)], "P0": 0}
        if len(head) == 1:                   # one frame: no pair; its window is itself, so its warp is the zoom
            with torch.cuda.device(dev):
                M = camera.stabilize_path([np.eye(3)], 0, 1, H, W, self.radius, self.crop)
                out = ops.warp_frames_affine(fr0.to(dev).unsqueeze(0).contiguous(), torch.from_numpy(M[None]).to(dev))
                res = out[0].cpu().numpy()
            yield res
            return
        yield from super().run(itertools.chain(head, it))
        with torch.cuda.device(dev):
            ready = self._warp_ready(len(self._v["P"]) + self._v["P0"])
        yield from ready


# ---------------------------------------------------------------------------------------------------------------------
# Moving-object segmentation
# ---------------------------------------------------------------------------------------------------------------------
class MotionFrame(NamedTuple):
    """The moving objects of one video frame.  labels (H,W) uint8: object k + 1 at the pixels of row k, 0 elsewhere;
    objects (count,10) float64 rows (area, x0, y0, x1, y1, cx, cy, peak, dx, dy) (ops.segment_motion); dropped: the
    objects found past max_objects, left unlabelled."""
    labels: np.ndarray
    objects: np.ndarray
    dropped: int


class VideoMotionSegmenter(VideoFlowPredictor):
    """The objects moving relative to the camera, streamed: run(frames) yields one MotionFrame per video frame, frame 0
    included, in order.

    The pairs go through VideoFlowPredictor's bidirectional machinery (frame buffer, pinned slots, copy streams, one CUDA
    graph per frame size and network.precision_key), and the graph continues after the occlusion masks with one
    ops.affine_motion(want_residual=True) over the batch's 2B flows and one ops.segment_motion over the batch's first B
    frames.  Frame t0 + j takes side a from pair j and side b from pair j - 1, or for j = 0 from a device copy of the
    previous batch's last backward residual and mask (NaN residuals at the start of a video: undefined).  The last
    frame is segmented from side b alone after the final batch.  Only the labels and the object rows cross PCIe; the
    padded tail of a partial batch is discarded.  The results equal network.segment_motion's bit for bit.  frames: host
    uint8 (H,W,3) arrays or tensors, any channel order."""

    def __init__(self, net: nn.Module, batch: int = 8, resize=None, tau_lo: float = ops.SEG_TAU_LO,
                 tau_hi: float = ops.SEG_TAU_HI, min_area: int = ops.SEG_MIN_AREA,
                 max_objects: int = ops.SEG_MAX_OBJECTS, alpha: float = 0.01, beta: float = 0.5, depth: int = 2):
        super().__init__(net, batch=batch, resize=resize, depth=depth, bidirectional=True, alpha=alpha, beta=beta)
        ops.check_segment_args(tau_lo, tau_hi, min_area, max_objects, "VideoMotionSegmenter")
        self.seg_args = dict(tau_lo=float(tau_lo), tau_hi=float(tau_hi), min_area=int(min_area),
                             max_objects=int(max_objects))
        self._carries = {}
        self._run = None          # (graph state, pairs of the last collected batch) of the video being run

    def invalidate(self) -> None:
        super().invalidate()
        self._carries.clear()

    def _carry(self, H: int, W: int, dev: torch.device):
        """The previous batch's last backward residual and mask, on the device."""
        c = self._carries.get((H, W))
        if c is None:
            c = self._carries[(H, W)] = {"res": torch.empty((1, H, W), dtype=torch.float32, device=dev),
                                         "occ": torch.empty((1, H, W), dtype=torch.uint8, device=dev)}
        return c

    def _chain(self, F: torch.Tensor, H: int, W: int):
        c = self._carry(H, W, F.device)
        flows = network._frame_pair_flows(self.net, F, self.resize, True)
        (labels, objects, count, dropped), res_bw, occ_bw = network._segment_batch(
            flows, (c["res"], c["occ"]), self.alpha, self.beta, self.seg_args)
        return {"labels": labels, "objects": objects, "count": count, "dropped": dropped, "res_bw": res_bw,
                "occ_bw": occ_bw}

    def _outputs(self):
        return ("labels", "objects", "count", "dropped")

    def _start(self, st) -> None:
        F = st["F"]
        c = self._carry(F.shape[1], F.shape[2], F.device)
        c["res"].fill_(float("nan"))
        c["occ"].zero_()
        self._run = (st, 0)

    def _collect(self, s, b: int) -> Iterator:
        self._run = (self._run[0], b)
        for labels, objects, count, dropped in super()._collect(s, b):
            yield MotionFrame(labels, objects[:int(count)], int(dropped))

    def _segment_last(self, res_bw, occ_bw, nb: int, shape) -> MotionFrame:
        labels, objects, count, dropped = network._segment_last(res_bw, occ_bw, nb, shape, self.seg_args)
        n = int(count[0])
        return MotionFrame(labels[0].cpu().numpy(), objects[0, :n].cpu().numpy(), int(dropped[0]))

    @torch.no_grad()
    def run(self, frames: Iterable) -> Iterator[MotionFrame]:
        it = iter(frames)
        head = [fr for fr in (next(it, None), next(it, None)) if fr is not None]
        if not head:
            return
        dev = next(self.net.parameters()).device
        if len(head) == 1:                   # one frame: no pair, an empty frame
            fr = self._frame(head[0], None)
            with torch.cuda.device(dev):
                yield self._segment_last(None, None, 0, (1, int(fr.shape[0]), int(fr.shape[1])))
            return
        yield from super().run(itertools.chain(head, it))
        st, b = self._run                    # the graph's outputs still hold the last batch
        self._run = None
        with torch.cuda.device(dev):
            yield self._segment_last(st["out"]["res_bw"], st["out"]["occ_bw"], b, None)


# ---------------------------------------------------------------------------------------------------------------------
# Video denoising
# ---------------------------------------------------------------------------------------------------------------------
class VideoDenoiser(_FrameRing, VideoFlowPredictor):
    """A denoised video, streamed: run(frames) yields one denoised (H,W,3) uint8 frame per input frame, frame 0 included,
    in order, `radius` frames behind the input.

    The pairs go through VideoFlowPredictor's bidirectional machinery (frame buffer, pinned slots, copy streams, one
    CUDA graph per frame size and network.precision_key); the graph ends at the 2B flows, and nothing of it comes back to
    the host.  On the compute stream each batch's new frames and both directions' flows are copied into a device ring of
    2 radius + depth * batch + 1 slots.  Once per collected batch, on a stream of its own, one ops.denoise_frames call
    denoises the frames whose window is complete (t + radius <= the last frame loaded); the last `radius` frames follow
    after the final batch, their windows clamped to the video.  sigma=None takes ops.median_noise of the first
    min(T, batch + 1) frames (the value used is left in `sigma_used`).  A one-frame video comes back unchanged.  Each
    frame crosses PCIe once in each direction, and memory is bounded by the radius and the batch, not the video's length.
    The results equal network.denoise_video's bit for bit.  frames: host uint8 (H,W,3) arrays or tensors, any channel
    order."""

    def __init__(self, net: nn.Module, batch: int = 8, resize=None, radius: int = ops.DENOISE_RADIUS, sigma=None,
                 h: float = ops.DENOISE_H, patch: int = ops.DENOISE_PATCH, alpha: float = 0.01, beta: float = 0.5,
                 depth: int = 2):
        super().__init__(net, batch=batch, resize=resize, depth=depth, bidirectional=True, alpha=alpha, beta=beta)
        ops.check_denoise_args(radius, sigma, h, patch, alpha, beta, "VideoDenoiser", sigma_optional=True)
        self.radius, self.h, self.patch = int(radius), float(h), int(patch)
        self.sigma = None if sigma is None else float(sigma)
        self.sigma_used = None
        self.ring_size = 2 * self.radius + self.depth * self.batch + 1
        self._rings = {}
        self._v = None          # the state of the video being run

    def invalidate(self) -> None:
        super().invalidate()
        self._rings.clear()

    def _chain(self, F: torch.Tensor, H: int, W: int):
        B = self.batch
        flows = network._frame_pair_flows(self.net, F, self.resize, True)
        return {"flow": flows[:B], "flow_bw": flows[B:]}

    def _outputs(self):
        return ()

    def _ring(self, H: int, W: int, dev: torch.device):
        """The device rings of frames and flows, the output buffers and the denoising stream."""
        e = self._rings.get((H, W))
        if e is None:
            n = self.ring_size
            e = self._rings[(H, W)] = {
                "frames": torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev),
                "fw": torch.empty((n, H, W, 2), dtype=torch.float32, device=dev),
                "bw": torch.empty((n, H, W, 2), dtype=torch.float32, device=dev),
                "out": torch.empty((n, H, W, 3), dtype=torch.uint8, device=dev),
                "out_host": torch.empty((n, H, W, 3), dtype=torch.uint8, pin_memory=True),
                "stream": torch.cuda.Stream(device=dev), "ev_done": torch.cuda.Event(), "ev_host": torch.cuda.Event(),
                "used": False}
        return e

    def _loaded(self, st, first: bool) -> None:
        """Copies the batch's new frames from the frame buffer into the ring, after the denoising that read their slots."""
        F = st["F"]
        v = self._v
        r = v["ring"]
        cur = torch.cuda.current_stream(F.device)
        if r["used"]:
            cur.wait_event(r["ev_done"])
        src = F if first else F[1:]
        t0 = v["loaded"]
        self._store(r["frames"], src, t0)
        v["pair0"] = 0 if first else t0 - 1          # the batch's pairs are pair0 .. pair0 + B - 1
        v["loaded"] += len(src)

    def _replayed(self, st) -> None:
        """Copies the batch's flows from the graph's outputs into the ring; the event marks the batch as loaded."""
        v = self._v
        r, out, p0 = v["ring"], st["out"], v["pair0"]
        self._store(r["fw"], out["flow"], p0)
        self._store(r["bw"], out["flow_bw"], p0)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(st["F"].device))
        v["marks"].append((p0, ev))

    def _denoise_ready(self, ev, t_end: int, t_hi: int) -> list:
        """Denoises frames next .. t_end of the video whose last frame so far is t_hi, and returns them on the host."""
        v = self._v
        t0 = v["next"]
        n = t_end - t0 + 1
        r = v["ring"]
        ws = r["stream"]
        if ev is not None:                   # also when nothing is ready: later calls rely on the stream's order
            ws.wait_event(ev)
        if n <= 0:
            return []
        with torch.cuda.stream(ws):
            ops.denoise_frames(r["frames"], r["fw"], r["bw"], self.radius, v["sigma"], self.h, self.patch, self.alpha,
                               self.beta, t0=t0, n=n, t_lo=0, t_hi=t_hi, out=r["out"][:n])
            r["ev_done"].record(ws)
            r["used"] = True
            r["out_host"][:n].copy_(r["out"][:n], non_blocking=True)
            r["ev_host"].record(ws)
        r["ev_host"].synchronize()
        v["next"] = t_end + 1
        return [r["out_host"][j].numpy().copy() for j in range(n)]

    def _collect(self, s, b: int) -> Iterator:
        p0, ev = self._v["marks"].popleft()
        last = p0 + b                                  # the batch's last real frame
        with torch.cuda.device(self._v["dev"]):
            ready = self._denoise_ready(ev, last - self.radius, last)
        yield from ready

    @torch.no_grad()
    def run(self, frames: Iterable) -> Iterator[np.ndarray]:
        it = iter(frames)
        head = list(itertools.islice(it, self.batch + 1))
        if not head:
            return
        fr0 = self._frame(head[0], None)
        H, W = int(fr0.shape[0]), int(fr0.shape[1])
        head = [fr0] + [self._frame(fr, (H, W)) for fr in head[1:]]
        dev = next(self.net.parameters()).device
        with torch.cuda.device(dev):
            sigma = self.sigma if self.sigma is not None else ops.median_noise(torch.stack(head).to(dev))
        self.sigma_used = sigma
        if len(head) == 1:                   # one frame: no neighbours
            yield head[0].numpy().copy()
            return
        count = [0]

        def counted(src):
            for fr in src:
                count[0] += 1
                yield fr

        with torch.cuda.device(dev):
            self._v = {"dev": dev, "ring": self._ring(H, W, dev), "loaded": 0, "next": 0, "pair0": 0,
                       "marks": collections.deque(), "sigma": sigma}
        yield from super().run(counted(itertools.chain(head, it)))
        with torch.cuda.device(dev):
            ready = self._denoise_ready(None, count[0] - 1, count[0] - 1)
        yield from ready
