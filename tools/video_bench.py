"""Video flow throughput with colour output (network.VideoFlowPredictor) and the time of the colour-coding kernel alone.

    python tools/video_bench.py [--hw 436x1024] [--resize 448,1024] [--batch 8] [--frames 65] [--host-frames 17]

All inputs are synthetic, from a seed.  Prints one JSON object with the card's name and power limit, read in the same run:
  video_fps[net]        frames/s host -> host: uint8 frames in, uint8 colour frames out, coloured on the GPU (one graph
                        replay per batch: HWC->NCHW, preprocess with resize, network, postprocess, mfn_flow_to_color)
  host_color_fps[net]   the same loop returning the float flow, coloured on the host by oracle/flowvis_ref.py (float64
                        numpy), which is how the reference colours a video (flow_vis on every flow)
  kernel[...]           mfn_flow_to_color alone at N=batch and the frame size, on a smooth and on a noise flow: CUDA
                        events over many launches replayed from a CUDA graph, the bytes
                        it must move (8 B/px read, 8 more for the per-sample max pass, 3 B/px written) over that time,
                        and the kernel's share of the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import network, ops  # noqa: E402
from maskflownet_b200.video import VideoFlowPredictor  # noqa: E402
from oracle import flowvis_ref  # noqa: E402

HBM_PEAK = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def video_rate(pred, frames, host_color):
    list(pred.run(frames[:2 * pred.batch + 1]))          # warm-up: graph capture, pinned staging
    torch.cuda.synchronize()
    t0, n = time.perf_counter(), 0
    for r in pred.run(frames):
        if host_color:
            flowvis_ref.flow_to_color(r[1])
        n += 1
    return n / (time.perf_counter() - t0)


def kernel_time(flow, max_radius, iters=100, replays=5):
    """Seconds per mfn_flow_to_color call, launched back to back from a CUDA graph so that the host's per-call cost does
    not enter (in per-sample mode a call is the memset, the max pass and the colour pass)."""
    ops.flow_to_color(flow, max_radius)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            ops.flow_to_color(flow, max_radius)
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        graph.replay()
    e1.record()
    e1.synchronize()
    t = e0.elapsed_time(e1) / 1e3 / (iters * replays)
    px = flow.numel() // 2
    nbytes = px * (8 + 3 + (8 if max_radius is None else 0))
    return {"us": round(t * 1e6, 2), "bytes": nbytes, "GB_s": round(nbytes / t / 1e9, 1),
            "kernel_share_of_hbm_peak": round(nbytes / t / HBM_PEAK, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hw", default="436x1024")
    ap.add_argument("--resize", default="448,1024")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--frames", type=int, default=65)
    ap.add_argument("--host-frames", type=int, default=17)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--precision", choices=("fp32", "bf16"), default="fp32", help="the models' inference_precision")
    a = ap.parse_args()
    H, W = map(int, a.hw.split("x"))
    resize = tuple(int(s) for s in a.resize.split(",")) if a.resize else None
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    rng = np.random.default_rng(a.seed)
    frames = rng.integers(0, 256, (a.frames, H, W, 3), dtype=np.uint8)
    res = {"gpu": gpu_info(), "hw": [H, W], "resize": resize, "batch": a.batch, "precision": a.precision, "video_fps": {},
           "host_color_fps": {}}
    for name, cls in (("MaskFlownet_S", network.MaskFlownetS), ("MaskFlownet", network.MaskFlownet)):
        torch.manual_seed(a.seed)
        model = cls().cuda().eval()
        model.inference_precision = a.precision
        res["video_fps"][name] = round(video_rate(VideoFlowPredictor(model, a.batch, resize), frames, False), 1)
        host = VideoFlowPredictor(model, a.batch, resize, want_flow=True)
        res["host_color_fps"][name] = round(video_rate(host, frames[:a.host_frames], True), 1)
        del model, host
        torch.cuda.empty_cache()
    # a smooth rotation (every angle, neighbouring pixels close on the wheel) and white noise (neighbours anywhere on it)
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    rot = np.stack([-(y - H / 2), x - W / 2], -1) * 0.05
    smooth = np.broadcast_to(rot, (a.batch, H, W, 2)) + rng.standard_normal((a.batch, H, W, 2)).astype(np.float32) * 0.1
    noise = rng.standard_normal((a.batch, H, W, 2)).astype(np.float32) * 10
    res["kernel"] = {}
    for fname, f in (("smooth", smooth), ("noise", noise)):
        t = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32)).cuda()
        res["kernel"][f"{fname}_per_sample"] = kernel_time(t, None)
        res["kernel"][f"{fname}_fixed_radius"] = kernel_time(t, 20.0)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
