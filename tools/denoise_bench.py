"""Video denoising cost on the GPU: the denoising kernel alone, and the video path against the plain predictor.

    python tools/denoise_bench.py [--iters 50] [--reps 3] [--frames 65] [--out results.json]

Kernel: ops.denoise_frames over a plain clip (S = N + 2R frames, the N middle ones denoised, every window full) at
N x H x W = 8 x 436 x 1024 and 2 x 1080 x 1920, R = 2 and R = 3, the default patch and h, timed with CUDA events over
`iters` calls after a warm-up.  The flows are a sub-pixel pan with noise, consistent in both directions, so every chain
runs its full length.  The algorithm gathers about 2R (2 x 8 + 3) + 3 B per output pixel (per chain step the two flow
samples and the colour) and writes 3 B; the halo of the tiles adds (16 + 2r)^2 / 16^2 of chain work.  The bytes are
given as a share of the H100 SXM's 3.35 TB/s of HBM3; the gathers mostly hit L2, so this is a scale, not a bound.
Noise estimate: ops.estimate_noise of 9 frames at each size.
Video: VideoDenoiser against VideoFlowPredictor(bidirectional=True), both MaskFlownet-S at batch 8 on 1024x436
synthetic frames, alternating in one process: input frames per second.
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
from maskflownet_b200.video import VideoDenoiser, VideoFlowPredictor  # noqa: E402

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


def bench_kernel(N, H, W, R, iters, dev):
    g = np.random.default_rng(0)
    S = N + 2 * R
    frames = torch.from_numpy(g.integers(0, 256, (S, H, W, 3), dtype=np.uint8)).to(dev)
    fw = torch.from_numpy((np.array([0.6, -0.3]) + g.normal(0, 0.05, (S, H, W, 2))).astype(np.float32)).to(dev)
    bw = -fw
    out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=dev)
    ms = _time(lambda: ops.denoise_frames(frames, fw, bw, R, 10.0, t0=R, n=N, out=out), iters)
    px = N * H * W
    nbytes = px * (2 * R * (2 * 8 + 3) + 3 + 3)
    sig_ms = _time(lambda: ops.estimate_noise(frames[:9] if S >= 9 else frames), iters)
    return {"N": N, "H": H, "W": W, "R": R, "patch": ops.DENOISE_PATCH, "ms": ms, "bytes": nbytes,
            "hbm_share": nbytes / HBM_BYTES_PER_S / (ms * 1e-3), "noise_frames": min(S, 9), "noise_ms": sig_ms}


def bench_video(model, frames, reps, batch):
    arms = {"VideoFlowPredictor": VideoFlowPredictor(model, batch=batch, bidirectional=True),
            "VideoDenoiser": VideoDenoiser(model, batch=batch, sigma=10.0)}
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
        raise SystemExit("denoise_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {"device": torch.cuda.get_device_properties(dev).name}
    try:
        out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                            "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        out["nvidia_smi"] = "not available"
    out["kernels"] = [bench_kernel(N, H, W, R, a.iters, dev) for N, H, W in ((8, 436, 1024), (2, 1080, 1920))
                      for R in (2, 3)]
    for r in out["kernels"]:
        print(f"{r['N']}x{r['H']}x{r['W']} R={r['R']}: denoise {r['ms']:.3f} ms ({r['hbm_share']:.2f} of HBM for "
              f"{r['bytes'] / 1e6:.1f} MB); noise estimate of {r['noise_frames']} frames {r['noise_ms']:.3f} ms")
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
