"""Kernel-level benchmark for the hot-path kernels at BASELINE config[1] shapes (batch 8, 1024x448, levels 6..2).

Times each kernel alone with CUDA events on the launching stream; between timed launches a 256 MiB buffer is
overwritten to flush the 50 MB L2 ("cold" numbers) unless --warm is given.  Prints one JSON object per line.
Development tool -- the reported numbers come from bench.py.

    python tools/kbench.py [--what corr,warp,bwd] [--iters 30] [--warm] [--n 8] [--hw 448x1024]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import ops, _lib  # noqa: E402

LEVELS = {6: 196, 5: 128, 4: 96, 3: 64, 2: 32}


def peaks():
    return 3350.0, "H100 SXM data sheet"


def timeit(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    tot = 0.0
    best = 1e9
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        # keep the GPU busy (~0.3 ms) while the CPU enqueues event + launch, so that the events bracket pure device
        # time and not the Python/ctypes launch latency
        torch.cuda._sleep(600_000)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        t = e0.elapsed_time(e1)
        tot += t
        best = min(best, t)
    return tot / iters, best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", default="corr,warp")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warm", action="store_true")
    ap.add_argument("--n", type=int, default=8)
    ap.add_argument("--hw", default="448x1024")
    ap.add_argument("--md", type=int, default=4)
    ap.add_argument("--levels", default="2,3,4,5,6")
    ap.add_argument("--algos", default="simt,mma_bf16x3,generic")
    args = ap.parse_args()
    H0, W0 = map(int, args.hw.split("x"))
    N = args.n
    what = args.what.split(",")
    dev = "cuda"
    peak, peak_kind = peaks()
    flush = None if args.warm else torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def emit(d):
        d.update({"N": N, "cold": not args.warm, "peak_gbs": peak, "peak_kind": peak_kind})
        s = json.dumps(d)
        print(s, flush=True)

    g = torch.Generator(device=dev).manual_seed(0)
    lv = [int(v) for v in args.levels.split(",")]
    for L, C in sorted(LEVELS.items()):
        if L not in lv:
            continue
        H, W = H0 >> L, W0 >> L
        f1 = torch.nn.functional.leaky_relu(torch.randn(N, C, H, W, device=dev, generator=g), 0.1)
        f2 = torch.nn.functional.leaky_relu(torch.randn(N, C, H, W, device=dev, generator=g), 0.1)
        md = args.md
        D = (2 * md + 1) ** 2
        if "corr" in what:
            nbytes = 4 * N * H * W * (2 * C + D)
            flops = 2 * D * C * N * H * W
            ref = None
            for name, algo in (("simt", ops.CORR_SIMT), ("mma_bf16x3", ops.CORR_MMA_BF16X3),
                               ("generic", ops.CORR_GENERIC)):
                if (algo == ops.CORR_GENERIC and L < 4) or name not in args.algos.split(","):
                    continue
                out = torch.empty(N, D, H, W, device=dev)
                fn = lambda: ops.correlation(f1, f2, pad_size=md, max_displacement=md, leaky_slope=0.1, algo=algo,
                                             out=out)
                try:
                    avg, best = timeit(fn, args.iters, flush)
                except Exception as e:  # noqa: BLE001
                    emit({"kernel": "corr_fwd", "algo": name, "level": L, "error": str(e)})
                    continue
                if ref is None:
                    ref = out.clone()
                    err = 0.0
                else:
                    err = (out - ref).abs().max().item()
                emit({"kernel": "corr_fwd", "algo": name, "launched": _lib.last_kernel(), "level": L, "C": C, "H": H,
                      "W": W, "ms_avg": round(avg, 5), "ms_best": round(best, 5), "alg_bytes": nbytes,
                      "gbs": round(nbytes / avg / 1e6, 1), "frac_of_peak": round(nbytes / avg / 1e6 / peak, 4),
                      "tflops_useful": round(flops / avg / 1e9, 2), "max_abs_diff_vs_first": err})
        if "warp" in what and L < 6:
            Fo = C
            w = torch.randn(Fo, C, 3, 3, device=dev, generator=g) * (2.0 / (9 * C)) ** 0.5
            b = torch.zeros(Fo, device=dev)
            flow_c = torch.randn(N, 2, H // 2, W // 2, device=dev, generator=g) * 0.4 * (2 ** L) / 20.0 / 4
            mask_c = torch.randn(N, 1, H // 2, W // 2, device=dev, generator=g) + 0.5
            trade = torch.randn(N, Fo, H, W, device=dev, generator=g) * 0.3
            packed = ops.conv3x3_pack(w)
            # the inference path of network.py: exact evaluation through linearity (warp_lin.cu)
            fn = lambda: ops.warp_mask(f2, flow_c, mask_c, w, b, trade, 20.0, float(2 ** L), 2, 0.1, 0,
                                       packed_weight=packed, resample=True)
            with torch.no_grad():
                avg, best = timeit(fn, args.iters, flush)
            nbytes = 4 * N * H * W * 3 * C + 4 * N * (H // 2) * (W // 2) * 3 + 4 * (9 * C * C + C)
            flops = 2 * 9 * C * C * N * H * W
            emit({"kernel": "warp_mask_fwd", "launched": _lib.last_kernel(), "level": L, "C": C, "H": H, "W": W,
                  "ms_avg": round(avg, 5), "ms_best": round(best, 5), "alg_bytes": nbytes,
                  "gbs": round(nbytes / avg / 1e6, 1), "frac_of_peak": round(nbytes / avg / 1e6 / peak, 4),
                  "tflops": round(flops / avg / 1e9, 2)})
        if "bwd" in what:
            go = torch.randn(N, D, H, W, device=dev, generator=g)
            t1, t2 = f1.clone().requires_grad_(), f2.clone().requires_grad_()
            out = ops.correlation(t1, t2, pad_size=md, max_displacement=md, leaky_slope=0.1, algo=ops.CORR_SIMT)

            def fn():
                t1.grad = t2.grad = None
                out.backward(go, retain_graph=True)
            avg, best = timeit(fn, max(3, args.iters // 3), flush)
            nbytes = 4 * N * H * W * (D + 4 * C)
            emit({"kernel": "corr_bwd", "level": L, "C": C, "ms_avg": round(avg, 5), "ms_best": round(best, 5),
                  "alg_bytes": nbytes, "gbs": round(nbytes / avg / 1e6, 1),
                  "frac_of_peak": round(nbytes / avg / 1e6 / peak, 4)})


if __name__ == "__main__":
    main()
