"""Kernel time of the deterministic backward entry points against their atomic counterparts (CUDA events, preallocated
buffers, the same inputs for both):

    python tools/det_bench.py [--iters 50]

  K4  mfn_warp_mask_backward(_det) at level 2 of BASELINE configs[2] (batch 8, 512x384: x (8,32,96,128), F = 32, mask)
  K5  mfn_image_warp_concat_backward(_det) at the cascade's shape (4,3,448,1024), all three gradients

Prints one JSON line per entry point: ms per call of each path, the ratio, and the device name and power limit.
"""
import argparse, json, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import ops


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    p = ops._p
    card = {"device": torch.cuda.get_device_name(dev), "power_limit": power_limit()}
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)

    # K4, level 2 of configs[2]
    N, C, F, H, W = 8, 32, 32, 96, 128
    x, w, b = rnd(N, C, H, W), rnd(F, C, 3, 3) * 0.08, rnd(F) * 0.1
    flow_c, mask_c, trade = rnd(N, 2, H // 2, W // 2) * 0.4, rnd(N, 1, H // 2, W // 2), rnd(N, F, H, W) * 0.3
    out, conv, fup, mup = (torch.empty(N, F, H, W, device=dev), torch.empty(N, F, H, W, device=dev),
                           torch.empty(N, 2, H, W, device=dev), torch.empty(N, 1, H, W, device=dev))
    ops._call("mfn_warp_mask_forward", dev, p(x), p(flow_c), p(mask_c), p(w), p(b), p(trade), p(out), p(fup), p(mup), p(conv),
              N, C, H, W, F, 2, 20.0, 4.0, 0.1, 0)
    go = rnd(N, F, H, W)
    gx, gf, gm, gw, gb, gt, ws = (torch.zeros_like(x), torch.empty_like(fup), torch.empty_like(mup), torch.zeros_like(w),
                                  torch.zeros_like(b), torch.empty_like(out), torch.empty_like(out))
    args = (p(go), p(out), p(conv), p(x), p(fup), p(mup), p(w), p(gx), p(gf), p(gm), p(gw), p(gb), p(gt), p(ws), N, C, H, W, F,
            20.0, 4.0, 0.1, 0)
    nb = ops.det_workspace_bytes("warp_mask", N, C, H, W, F)
    det_ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    t_atomic = timed(lambda: ops._call("mfn_warp_mask_backward", dev, *args), a.iters)
    t_det = timed(lambda: ops._call("mfn_warp_mask_backward_det", dev, *args, p(det_ws), nb), a.iters)
    print(json.dumps({"bench": "k4_backward_level2", "shape": [N, C, F, H, W], "atomic_ms": round(t_atomic, 4),
                      "det_ms": round(t_det, 4), "det_over_atomic": round(t_det / t_atomic, 3),
                      "det_ws_mb": round(nb / 1e6, 1), **card}))

    # K5 at the cascade's input shape
    N, Ci, H, W = 4, 3, 448, 1024
    im2, fq, mq, g40 = rnd(N, Ci, H, W), rnd(N, 2, H // 4, W // 4), rnd(N, 1, H // 4, W // 4), rnd(N, Ci + 1, H, W)
    gi2, gfu, gmu = torch.zeros_like(im2), torch.empty(N, 2, H, W, device=dev), torch.empty(N, 1, H, W, device=dev)
    args = (p(g40), p(im2), p(fq), p(mq), p(gi2), p(gfu), p(gmu), N, Ci, H, W, 20.0)
    nb = ops.det_workspace_bytes("image_warp_concat", N, Ci, H, W)
    det_ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    t_atomic = timed(lambda: ops._call("mfn_image_warp_concat_backward", dev, *args), a.iters)
    t_det = timed(lambda: ops._call("mfn_image_warp_concat_backward_det", dev, *args, p(det_ws), nb), a.iters)
    print(json.dumps({"bench": "k5_backward", "shape": [N, Ci, H, W], "atomic_ms": round(t_atomic, 4),
                      "det_ms": round(t_det, 4), "det_over_atomic": round(t_det / t_atomic, 3),
                      "det_ws_mb": round(nb / 1e6, 1), **card}))


if __name__ == "__main__":
    main()
