"""Video stabilisation cost on the GPU: the fit and the warp kernels alone, and the video path against the plain predictor.

    python tools/stabilize_bench.py [--iters 50] [--reps 3] [--frames 65] [--out results.json]

Kernels: ops.affine_motion (at the default iterations I) and ops.warp_frames_affine at N = 8 for 436x1024 and 1080x1920,
timed with CUDA events over `iters` calls after a warm-up.  The algorithm moves I N H W 8 B for the fit (the flow read
once per iteration) and 6 N H W B for the warp (3 B read, 3 B written per pixel); each is given as a share of the
H100 SXM's 3.35 TB/s of HBM3.  At 436x1024 the batch's flow (29 MB) fits in the 50 MB L2, so the fit's iterations after
the first may read it from L2, faster than HBM allows: a share above 1 says so.
Video: VideoStabilizer against VideoFlowPredictor (one direction, colour output only as its graph produces it), both
MaskFlownet-S at batch 8 on 1024x436 synthetic frames, alternating in one process: input frames per second.
"""
from __future__ import annotations

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
from maskflownet_b200.video import VideoFlowPredictor, VideoStabilizer  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _time(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_kernels(N, H, W, iters, dev):
    g = np.random.default_rng(0)
    y, x = np.mgrid[0:H, 0:W].astype(np.float32)
    flow = np.stack([0.01 * y + 2.0 + g.normal(0, 0.5, (N, H, W)), -0.01 * x + 1.0 + g.normal(0, 0.5, (N, H, W))], -1)
    flow = torch.from_numpy(flow.astype(np.float32)).to(dev)
    frames = torch.from_numpy(g.integers(0, 256, (N, H, W, 3), dtype=np.uint8)).to(dev)
    M = torch.tensor([[[0.99, 0.02, 5.0], [-0.02, 0.99, -3.0]]] * N, dtype=torch.float64, device=dev)
    I = ops.AFFINE_ITERATIONS
    fit_ms = _time(lambda: ops.affine_motion(flow, I), iters)
    warp_ms = _time(lambda: ops.warp_frames_affine(frames, M), iters)
    px = N * H * W
    fit_bytes, warp_bytes = I * px * 8, 6 * px
    return {"N": N, "H": H, "W": W, "iterations": I, "fit_ms": fit_ms, "fit_ms_per_iteration": fit_ms / I,
            "fit_bytes": fit_bytes, "fit_hbm_share": fit_bytes / HBM_BYTES_PER_S / (fit_ms * 1e-3),
            "warp_ms": warp_ms, "warp_bytes": warp_bytes, "warp_hbm_share": warp_bytes / HBM_BYTES_PER_S / (warp_ms * 1e-3)}


def bench_video(model, frames, reps, batch):
    arms = {"VideoFlowPredictor": VideoFlowPredictor(model, batch=batch), "VideoStabilizer": VideoStabilizer(model,
                                                                                                             batch=batch)}
    for p in arms.values():                       # capture the graphs outside the timed runs
        list(p.run(frames[:batch + 1]))
    res = {k: [] for k in arms}
    for _ in range(reps):
        for k, p in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = sum(1 for _ in p.run(frames))
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert n == len(frames) - (1 if k == "VideoFlowPredictor" else 0)
            res[k].append({"s": dt, "frames_per_s": len(frames) / dt})
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=65)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("stabilize_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {"device": torch.cuda.get_device_properties(dev).name}
    try:
        out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                            "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        out["nvidia_smi"] = "not available"
    out["kernels"] = [bench_kernels(8, H, W, a.iters, dev) for H, W in ((436, 1024), (1080, 1920))]
    for r in out["kernels"]:
        print(f"{r['N']}x{r['H']}x{r['W']}: fit {r['fit_ms']:.3f} ms ({r['fit_ms_per_iteration']:.4f} ms per iteration, "
              f"{r['fit_hbm_share']:.2f} of HBM), warp {r['warp_ms']:.3f} ms ({r['warp_hbm_share']:.2f} of HBM)")
    torch.manual_seed(0)
    model = network.MaskFlownetS().to(dev).eval()
    g = np.random.default_rng(1)
    frames = list(g.integers(0, 256, (a.frames, 436, 1024, 3), dtype=np.uint8))
    out["video"] = bench_video(model, frames, a.reps, 8)
    for k, runs in out["video"].items():
        print(f"video {k}: frames/s " + " ".join(f"{r['frames_per_s']:.1f}" for r in runs))
    print(out["nvidia_smi"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
