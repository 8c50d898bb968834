"""What unsupervised fine-tuning costs on the GPU.

    python tools/unsup_bench.py [--rounds 5] [--steps 5] [--warmup 3] [--kernel-iters 50] [--json FILE]

1. ms per step of PipelineFlownet.train_batch_unsupervised against train_batch at the same shape, in alternating rounds
   (each round: --steps steps of one, then of the other; CUDA events around each run of steps, which ends in a
   synchronise), for MaskFlownet-S with 4 pairs at 384x512 and the cascade with its head frozen (fix_head) with 4 pairs
   at 320x768.  Both steps use the same colour augmentation; train_batch also its geometric augmentation and a random
   label.  The unsupervised step runs the network at batch 2n (both directions of each pair).
2. each loss kernel alone at 2N = 8, 384x512 (the loss shape of the first configuration): CUDA events over
   --kernel-iters launches, the algorithmic bytes and flops from the shape (per pixel, counted from the source of
   csrc/unsup_loss.cu), and its share of the larger of the two H100 SXM data-sheet bounds (3.35 TB/s HBM3, 67 TFLOP/s
   FP32 non-tensor).
3. the card's name and power limit, read in the same run.
Prints one JSON object.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import augment, ops, pipeline  # noqa: E402

HBM_BPS, FP32_FLOPS = 3.35e12, 67e12
# per pixel of the (2N,H,W) loss shape: (bytes, flops)
#   census forward:  two RGB images and occ read, coef written; grey 2 x 6, per offset 2 x t (5) + s, phi and the sum (5)
#   census backward: two RGB images and coef read, the RGB gradient written; per offset ~23 operations
#   smoothness forward:  flow and image read; per direction one edge weight (~12) and two channels (~5 each)
#   smoothness backward: flow and image read, the flow gradient written; 6 edge weights, 12 second differences and signs
KERNEL_COST = {"census_forward": (4 * 6 + 1 + 4, 2 * 6 + 48 * 15 + 12),
               "census_backward": (4 * 6 + 4 + 4 * 3, 48 * 23 + 6),
               "smoothness_forward": (4 * 2 + 4 * 3, 2 * (12 + 2 * 5)),
               "smoothness_backward": (4 * 2 + 4 * 3 + 4 * 2, 6 * 12 + 12 * 5 + 8)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.TimeoutExpired):
        out = []
    return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()


def timed(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def step_comparison(network_class, n, shape, rounds, steps, warmup, fix_head=False):
    H, W = shape
    torch.manual_seed(0)
    pipe = pipeline.PipelineFlownet(network_class=network_class)
    if fix_head:
        pipe.fix_head()
    rng = np.random.default_rng(0)
    img1 = rng.integers(0, 256, (n, 3, H, W), dtype=np.uint8)
    img2 = np.roll(img1, (3, -5), axis=(2, 3))
    label = (rng.standard_normal((n, 2, H, W)) * 2).astype(np.float32)
    geo = augment.GeometryAugmentation(angle_range=(-17, 17), zoom_range=(0.9, 1 / 0.9), aspect_range=(0.95, 1 / 0.95),
                                       translation_range=0.05, target_shape=shape, orig_shape=shape, batch_size=n,
                                       relative_angle=0.25, relative_scale=(0.96, 1 / 0.96), relative_translation=0.25, seed=3)
    col = augment.ColorAugmentation(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4), batch_size=n,
                                    shape=shape, noise_range=(0, 0), saturation=0.5, hue=0.5, seed=4)
    sup = lambda: pipe.train_batch(img1, img2, label, geo, col)  # noqa: E731
    uns = lambda: pipe.train_batch_unsupervised(img1, img2, color_aug=col)  # noqa: E731
    for _ in range(warmup):
        sup()
        uns()
    t_sup, t_uns = [], []
    for _ in range(rounds):
        t_sup.append(timed(sup, steps))
        t_uns.append(timed(uns, steps))
    return {"network": network_class + (" (head frozen)" if fix_head else ""), "pairs": n, "shape": [H, W],
            "train_batch_ms": [round(t, 2) for t in t_sup], "train_batch_unsupervised_ms": [round(t, 2) for t in t_uns],
            "median_ratio": round(float(np.median(t_uns) / np.median(t_sup)), 3)}


def kernel_times(N, H, W, iters):
    rng = np.random.default_rng(1)
    dev = torch.device("cuda")
    img1 = torch.from_numpy(rng.random((N, 3, H, W), dtype=np.float32)).to(dev)
    img2 = torch.from_numpy(rng.random((N, 3, H, W), dtype=np.float32)).to(dev)
    occ = torch.from_numpy((rng.random((N, H, W)) < 0.1).astype(np.uint8)).to(dev)
    flow = torch.from_numpy(rng.standard_normal((N, 2, H, W), dtype=np.float32)).to(dev)
    g = torch.ones(N, device=dev)
    _, vsum, coef = ops._census_forward(img1, img2, occ)
    calls = {"census_forward": lambda: ops._census_forward(img1, img2, occ),
             "census_backward": lambda: ops._census_backward(img1, img2, coef, vsum, g),
             "smoothness_forward": lambda: ops._smoothness_forward(flow, img1),
             "smoothness_backward": lambda: ops._smoothness_backward(flow, img1, g)}
    out, px = {}, N * H * W
    for name, fn in calls.items():
        timed(fn, 3)
        ms = timed(fn, iters)
        b, f = KERNEL_COST[name]
        bound_s = max(px * b / HBM_BPS, px * f / FP32_FLOPS)
        out[name] = {"ms": round(ms, 4), "bytes": px * b, "flops": px * f,
                     "bound": "flops" if px * f / FP32_FLOPS > px * b / HBM_BPS else "bytes",
                     "share_of_bound": round(bound_s * 1e3 / ms, 3)}
    out["total_ms"] = round(sum(v["ms"] for v in out.values()), 4)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("unsup_bench.py measures on the GPU; no CUDA device found")
    res = {"card": card(),
           "steps": [step_comparison("MaskFlownet_S", 4, (384, 512), a.rounds, a.steps, a.warmup),
                     step_comparison("MaskFlownet", 4, (320, 768), a.rounds, a.steps, a.warmup, fix_head=True)],
           "loss_kernels_2N8_384x512": kernel_times(8, 384, 512, a.kernel_iters)}
    s = res["steps"][0]
    res["loss_kernels_share_of_unsupervised_step"] = round(
        res["loss_kernels_2N8_384x512"]["total_ms"] / float(np.median(s["train_batch_unsupervised_ms"])), 4)
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
