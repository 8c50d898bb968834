"""Dense point tracking cost on the GPU: the tracking launches alone, and the video tracker against the bidirectional video
predictor it extends.

    python tools/track_bench.py [--iters 50] [--rounds 3] [--frames 65] [--out results.json]

Launches: per frame, ops.track_advance (a memset of the cell map and one thread per slot) and ops.track_seed (one CTA:
query births and the block scans), plus the texture of the batch's frames (one thread per seed point and frame, timed
per frame as 1/N of one launch over N + 1 = 9 frames), at 8 x 436 x 1024 and 1 x 1080 x 1920 with spacing 8 and 4,
timed with CUDA events over `iters` repetitions after a warm-up.  The state is the default capacity (2 Gx Gy dense
slots) filled by a first frame; the flows are a smooth random field of a few pixels, so most tracks stay alive.
Video: VideoTracker against VideoFlowPredictor(bidirectional=True), both MaskFlownet-S at batch 8 on synthetic
1024 x 436 frames, in alternating rounds in one process: frames per second.
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
from maskflownet_b200.video import VideoFlowPredictor, VideoTracker  # noqa: E402


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name()


def _smooth_flow(rng, H, W, scale=3.0):
    from scipy.ndimage import gaussian_filter
    f = np.stack([gaussian_filter(rng.standard_normal((H // 8 + 1, W // 8 + 1)), 2) for _ in range(2)], -1)
    f = f / np.abs(f).max() * scale
    f = np.kron(f, np.ones((8, 8, 1)))[:H, :W]
    return torch.from_numpy(f.astype(np.float32)).cuda()


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench_launches(N, H, W, h, iters):
    rng = np.random.default_rng(0)
    frames = torch.from_numpy(rng.integers(0, 256, (N + 1, H, W, 3), dtype=np.uint8)).cuda()
    fw = _smooth_flow(rng, H, W)
    bw = -fw
    st = ops.TrackState(H, W, spacing=h)
    lam, lmax = ops.track_texture(frames, h)
    ops.track_start(st, frames[0])
    xy = torch.empty((st.K, 2), device="cuda")
    status = torch.empty((st.K,), dtype=torch.uint8, device="cuda")
    t_tex = _time(lambda: ops.track_texture(frames, h), iters) / (N + 1)
    t_adv = _time(lambda: ops.track_advance(st, fw, bw), iters)
    t_seed = _time(lambda: ops.track_seed(st, lam[1], lmax[1:2], xy, status), iters)
    alive = int(((status == ops.TRACK_TRACKED) | (status == ops.TRACK_BORN)).sum())
    return {"N": N, "H": H, "W": W, "spacing": h, "slots": st.K, "cells": st.Gx * st.Gy, "alive": alive,
            "texture_ms_per_frame": t_tex, "advance_ms": t_adv, "seed_ms": t_seed,
            "per_frame_ms": t_tex + t_adv + t_seed, "per_batch_ms": N * (t_tex + t_adv + t_seed)}


def bench_video(frames, rounds):
    torch.manual_seed(0)
    model = network.MaskFlownetS().cuda().eval()
    arms = {"bidirectional": VideoFlowPredictor(model, batch=8, bidirectional=True),
            "tracker": VideoTracker(model, batch=8)}
    for p in arms.values():                   # capture and warm up
        for _ in p.run(iter(frames[:17])):
            pass
    res = {k: [] for k in arms}
    for _ in range(rounds):
        for name, p in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = sum(1 for _ in p.run(iter(frames)))
            torch.cuda.synchronize()
            res[name].append(len(frames) / (time.perf_counter() - t0))
            assert n == len(frames) - (name == "bidirectional")
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=65)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "track_bench.py needs a GPU"
    out = {"gpu": _gpu_info(), "launches": [], "video": None}
    print(out["gpu"])
    for N, H, W in ((8, 436, 1024), (1, 1080, 1920)):
        for h in (8, 4):
            r = bench_launches(N, H, W, h, a.iters)
            out["launches"].append(r)
            print(f"{N}x{H}x{W} spacing {h}: {r['slots']} slots, {r['alive']} alive; texture {r['texture_ms_per_frame']:.4f}"
                  f" ms/frame, advance {r['advance_ms']:.4f} ms, seed {r['seed_ms']:.4f} ms; per frame "
                  f"{r['per_frame_ms']:.4f} ms, per batch of {N} {r['per_batch_ms']:.3f} ms")
    rng = np.random.default_rng(1)
    frames = [rng.integers(0, 256, (436, 1024, 3), dtype=np.uint8) for _ in range(a.frames)]
    v = bench_video(frames, a.rounds)
    out["video"] = v
    for k, fps in v.items():
        print(f"video {k}: " + ", ".join(f"{x:.1f}" for x in fps) + " frames/s")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
