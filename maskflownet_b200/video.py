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
Copies follow network.PipelinedFlowPredictor's slot scheme: pinned host staging, H2D on one copy stream, D2H of the colours
(and flows) on another, `depth` slots, so the copies of neighbouring batches run under the replay of this one.
"""
from __future__ import annotations

import collections
from typing import Iterable, Iterator

import numpy as np
import torch
import torch.nn as nn

from . import network, ops
from ._lib import MaskflowError

_WARMUP = 2


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
        x = F.permute(0, 3, 1, 2).contiguous()
        a, b, _ = ops.preprocess(x[:B], x[1:], ops.padded_size(H, W, self.resize))
        if not self.bidirectional:
            flow = ops.postprocess(self.net(a, b)[0][-1], H, W, flip_channels=True, is_flow=True)
            rgb, _ = ops.flow_to_color(flow, self.max_radius, self.bgr)
            return {"rgb": rgb, "flow": flow}
        flows = ops.postprocess(self.net(a, b, bidirectional=True)[0][-1], H, W, flip_channels=True, is_flow=True)
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
        else:
            F[0].copy_(F[B])
            F[1:].copy_(s["in"][:B])
        s["ev_in_free"].record(cur)
        st["graph"].replay()
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
