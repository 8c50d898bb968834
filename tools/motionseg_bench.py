"""Moving-object segmentation cost on the GPU: the segment call alone, and the video path against the bidirectional
predictor.

    python tools/motionseg_bench.py [--iters 50] [--reps 3] [--frames 65] [--out results.json]

Kernel: ops.segment_motion at N = 8 for 436x1024 and 1080x1920, timed with CUDA events over `iters` calls after a
warm-up, on two inputs: the synthetic scene's residuals (a panning, rotating, zooming camera with two moving objects,
tests/test_motion_segment.py) and noise at density 0.41, near the 8-neighbour site-percolation threshold, where
components are largest and most tangled (the worst case for the union-find).  The algorithm reads 18 B per pixel once
(two residuals, two masks, the forward flow) and writes 1 B of labels; the call's launches read them twice and move
the 4 B parent array a few times more, so the share of the H100 SXM's 3.35 TB/s given here is of the 19 B per pixel
the algorithm needs.  Also the workspace bytes.
Video: VideoMotionSegmenter against VideoFlowPredictor(bidirectional=True), both MaskFlownet-S at batch 8 on 1024x436
synthetic frames, alternating in one process: input frames per second of each round.
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
from maskflownet_b200 import _lib, network, ops  # noqa: E402
from maskflownet_b200.video import VideoFlowPredictor, VideoMotionSegmenter  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BYTES_PER_PIXEL = 4 + 1 + 4 + 1 + 8 + 1


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


def _camera(H, W, pan, deg, zoom):
    c, s = zoom * np.cos(np.radians(deg)), zoom * np.sin(np.radians(deg))
    L = np.array([[c, -s], [s, c]])
    ctr = np.array([(W - 1) / 2, (H - 1) / 2])
    return np.concatenate([L, (ctr - L @ ctr + np.array(pan))[:, None]], 1)


def scene_inputs(N, H, W, dev, g):
    """The synthetic scene's inputs: per frame, the camera's flow both ways with 0.3 px noise and a square and a disc
    moving 6 px and 3 px relative to it; residuals and fits from ops.affine_motion."""
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    sq = (np.abs(x - 0.3 * W) <= 0.1 * min(H, W)) & (np.abs(y - 0.35 * H) <= 0.1 * min(H, W))
    di = (x - 0.7 * W) ** 2 + (y - 0.6 * H) ** 2 <= (0.12 * min(H, W)) ** 2
    flows = np.empty((2 * N, H, W, 2), np.float32)
    for n in range(N):
        A = _camera(H, W, g.uniform(-6, 6, 2), g.uniform(-1, 1), g.uniform(0.98, 1.02))
        L = np.linalg.inv(A[:, :2])
        Ab = np.concatenate([L, -(L @ A[:, 2])[:, None]], 1)
        for k, (M, sign) in enumerate(((A, 1.0), (Ab, -1.0))):
            f = np.stack([M[0, 0] * x + M[0, 1] * y + M[0, 2] - x, M[1, 0] * x + M[1, 1] * y + M[1, 2] - y], -1)
            f[sq] += sign * np.array([4.8, -3.6])
            f[di] += sign * np.array([0.0, 3.0])
            flows[k * N + n] = f + g.normal(0, 0.3, f.shape)
    fl = torch.from_numpy(flows).to(dev)
    affine, _, res = ops.affine_motion(fl, want_residual=True)
    occ = torch.zeros((N, H, W), dtype=torch.uint8, device=dev)
    return res[:N].contiguous(), occ, res[N:].contiguous(), occ, fl[:N].contiguous(), affine[:N].contiguous()


def noise_inputs(N, H, W, dev, g, density=0.41):
    m = g.random((2, N, H, W)) < density
    r = torch.from_numpy(np.where(m, 3.0, 0.0).astype(np.float32)).to(dev)
    occ = torch.zeros((N, H, W), dtype=torch.uint8, device=dev)
    flow = torch.from_numpy(g.normal(0, 2, (N, H, W, 2)).astype(np.float32)).to(dev)
    A = torch.tensor([[[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]] * N, dtype=torch.float64, device=dev)
    # the same mask on both sides, so s keeps the percolation density
    return r[0], occ, r[0].clone(), occ, flow, A


def bench_kernel(N, H, W, iters, dev):
    g = np.random.default_rng(0)
    px = N * H * W
    out = {"N": N, "H": H, "W": W, "workspace_bytes": int(_lib.lib().mfn_motion_segment_workspace_bytes(N, H, W)),
           "algorithm_bytes": BYTES_PER_PIXEL * px}
    for name, inputs in (("scene", scene_inputs(N, H, W, dev, g)), ("noise_0.41", noise_inputs(N, H, W, dev, g))):
        kw = dict(min_area=1) if name.startswith("noise") else {}
        _, _, count, dropped = ops.segment_motion(*inputs, **kw)
        ms = _time(lambda: ops.segment_motion(*inputs, **kw), iters)
        out[name] = {"ms": ms, "hbm_share": BYTES_PER_PIXEL * px / HBM_BYTES_PER_S / (ms * 1e-3),
                     "count": count.tolist(), "dropped": dropped.tolist()}
    return out


def bench_video(model, frames, reps, batch):
    arms = {"VideoFlowPredictor(bidirectional)": VideoFlowPredictor(model, batch=batch, bidirectional=True),
            "VideoMotionSegmenter": VideoMotionSegmenter(model, batch=batch)}
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
            assert n == len(frames) - (1 if k.startswith("VideoFlowPredictor") else 0)
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
        raise SystemExit("motionseg_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    out = {"device": torch.cuda.get_device_properties(dev).name}
    try:
        out["nvidia_smi"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                            "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        out["nvidia_smi"] = "not available"
    out["kernel"] = [bench_kernel(8, H, W, a.iters, dev) for H, W in ((436, 1024), (1080, 1920))]
    for r in out["kernel"]:
        print(f"{r['N']}x{r['H']}x{r['W']}: workspace {r['workspace_bytes'] / 2**20:.1f} MiB; " + "; ".join(
            f"{k} {r[k]['ms']:.3f} ms ({r[k]['hbm_share']:.2f} of HBM for {BYTES_PER_PIXEL} B/px)"
            for k in ("scene", "noise_0.41")))
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
