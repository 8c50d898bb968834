"""Forward throughput of the two inference precisions, measured in one process with the precisions alternating.

    python tools/precision_bench.py [--batch 8] [--height 448] [--width 1024] [--steps 20] [--warmup 3] [--rounds 5]
                                    [--json FILE]

bench.py's method at bench.py's default shape: random-init (MSRAPrelu, seed 0) MaskFlownet-S and the cascade, batch 8,
1024x448 synthetic uint8 pairs already on the device, one network.FlowPredictor CUDA-graph replay per step, a 256 MiB
buffer overwritten before every step (inside the timed region, so every step starts with a cold L2), CUDA events around
--steps steps.  Each model is timed in --rounds rounds; a round times fp32 then bf16 (inference_precision), so that
clock and load drift fall on both alike.  Prints pairs/s per round and the median per precision, with the card's name,
its power limit and its maximum SM clock (nvidia-smi), and the median bf16 / fp32 ratio.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import network  # noqa: E402

PRECISIONS = ("fp32", "bf16")


def gpu_info() -> dict:
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, plim, cmax, cur = (s.strip() for s in out[torch.cuda.current_device()].split(","))
        return {"name": name, "power_limit": plim, "sm_clock_max": cmax, "sm_clock_idle": cur}
    except Exception as e:   # nvidia-smi missing: the device name from torch, the rest unknown
        return {"name": torch.cuda.get_device_name(), "error": str(e)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=448)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("precision_bench.py times the GPU forward: no CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    g = torch.Generator().manual_seed(100)
    shape = (a.batch, 3, a.height, a.width)
    im1 = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g).to(dev)
    im2 = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g).to(dev)
    res = {"gpu": gpu_info(), "batch": a.batch, "hw": [a.height, a.width], "steps": a.steps, "rounds": a.rounds,
           "method": "FlowPredictor graph replay, 256 MiB L2 flush before every step, CUDA events", "models": {}}

    def timed(pred):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            flush.zero_()
            pred(im1, im2)
        e1.record()
        torch.cuda.synchronize()
        return a.batch * a.steps / (e0.elapsed_time(e1) * 1e-3)

    for name, cls in (("MaskFlownet_S", network.MaskFlownetS), ("MaskFlownet", network.MaskFlownet)):
        torch.manual_seed(0)
        model = cls().to(dev).eval()
        pred = network.FlowPredictor(model)
        rates = {p: [] for p in PRECISIONS}
        with torch.no_grad():
            for p in PRECISIONS:                              # capture both graphs and warm up
                model.inference_precision = p
                for _ in range(a.warmup):
                    pred(im1, im2)
            for r in range(a.rounds):
                for p in PRECISIONS:
                    model.inference_precision = p
                    rates[p].append(timed(pred))
                print(f"{name} round {r}: " + ", ".join(f"{p} {rates[p][-1]:.1f} pairs/s" for p in PRECISIONS), flush=True)
        med = {p: statistics.median(v) for p, v in rates.items()}
        res["models"][name] = {"pairs_per_s": {p: round(med[p], 2) for p in PRECISIONS},
                               "rounds": {p: [round(x, 2) for x in v] for p, v in rates.items()},
                               "bf16_over_fp32": round(med["bf16"] / med["fp32"], 3)}
        print(f"{name}: median fp32 {med['fp32']:.1f}, bf16 {med['bf16']:.1f} pairs/s, x{med['bf16'] / med['fp32']:.3f}")
        del model, pred
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
