"""Frame interpolation cost on the GPU: the splatting kernels alone, and the video path with and without interpolation.

    python tools/interp_bench.py [--iters 20] [--reps 3] [--frames 65] [--out results.json]

Kernel: ops.interpolate_frames at N = 8 for 436x1024 and 1080x1920, T = 1 and 7, timed with CUDA events over `iters`
calls after a warm-up.  Per time step each source pixel issues at most 16 int64 atomics (4 corners x 4 sums); the
algorithmic bytes per step are the inputs read once (2 x (3 + 8 + 1) B per pixel), the workspace zeroed and read back
(2 x 32 B) and the output slice written (3 B).  The flows are a smooth random field of a few pixels, like network flows.
Video: VideoFlowPredictor(MaskFlownet-S, batch 8) on 1024x436 synthetic frames, bidirectional without interpolation
against interpolate=1 and interpolate=7, alternating in one process: pairs per second and output frames per second
(one colour image per pair, or T in-between frames plus the pair's second frame).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import network, ops  # noqa: E402
from maskflownet_b200.video import VideoFlowPredictor  # noqa: E402


def _smooth_flow(g, N, H, W, amp, dev):
    coarse = torch.from_numpy(g.normal(0, amp, (N, 2, H // 32 + 2, W // 32 + 2)).astype(np.float32)).to(dev)
    f = torch.nn.functional.interpolate(coarse, size=(H, W), mode="bicubic", align_corners=False)
    return f.permute(0, 2, 3, 1).contiguous()


def bench_kernel(N, H, W, T, iters, dev):
    g = np.random.default_rng(0)
    img0, img1 = (torch.from_numpy(g.integers(0, 256, (N, H, W, 3), dtype=np.uint8)).to(dev) for _ in range(2))
    fw = _smooth_flow(g, N, H, W, 4.0, dev)
    bw = -fw
    ofw, obw = ops.flow_consistency(fw, bw)
    times = [k / (T + 1) for k in range(1, T + 1)]
    for _ in range(3):
        ops.interpolate_frames(img0, img1, fw, bw, ofw, obw, times)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.interpolate_frames(img0, img1, fw, bw, ofw, obw, times)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    px = N * H * W
    step_bytes = px * (2 * (3 + 8 + 1) + 2 * 32 + 3)
    atomics = 16 * 2 * px
    return {"N": N, "H": H, "W": W, "T": T, "ms_per_call": ms, "ms_per_step": ms / T,
            "atomics_per_step": atomics, "gatomics_per_s": atomics * T / ms / 1e6,
            "algorithmic_bytes_per_step": step_bytes, "algorithmic_gb_per_s": step_bytes * T / ms / 1e6}


def bench_video(model, frames, reps, batch):
    arms = {"bidirectional": dict(bidirectional=True), "interpolate=1": dict(interpolate=1),
            "interpolate=7": dict(interpolate=7)}
    preds = {k: VideoFlowPredictor(model, batch=batch, **kw) for k, kw in arms.items()}
    for p in preds.values():                       # capture the graphs outside the timed runs
        list(p.run(frames[:batch + 1]))
    pairs = len(frames) - 1
    res = {k: [] for k in arms}
    for _ in range(reps):
        for k, p in preds.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = sum(1 for _ in p.run(frames))
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert n == pairs
            T = p.interpolate
            res[k].append({"s": dt, "pairs_per_s": pairs / dt, "out_frames_per_s": pairs * (T + 1 if T else 1) / dt})
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=65)
    ap.add_argument("--out", default=None, help="also write the results as JSON to this path")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("interp_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    out = {"device": props.name}
    try:
        import subprocess
        out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                            "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        out["nvidia_smi"] = "not available"
    out["kernel"] = [bench_kernel(8, H, W, T, a.iters, dev) for H, W in ((436, 1024), (1080, 1920)) for T in (1, 7)]
    for r in out["kernel"]:
        print(f"kernel {r['N']}x{r['H']}x{r['W']} T={r['T']}: {r['ms_per_call']:.3f} ms per call, {r['ms_per_step']:.3f} ms "
              f"per step, {r['gatomics_per_s']:.1f} G atomics/s, {r['algorithmic_gb_per_s']:.0f} GB/s algorithmic")
    torch.manual_seed(0)
    model = network.MaskFlownetS().to(dev).eval()
    g = np.random.default_rng(1)
    frames = list(g.integers(0, 256, (a.frames, 436, 1024, 3), dtype=np.uint8))
    out["video"] = bench_video(model, frames, a.reps, 8)
    for k, runs in out["video"].items():
        print(f"video {k}: pairs/s " + " ".join(f"{r['pairs_per_s']:.1f}" for r in runs) + "; output frames/s " +
              " ".join(f"{r['out_frames_per_s']:.1f}" for r in runs))
    print(out["nvidia_smi"])
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
