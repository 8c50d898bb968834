"""How much the bf16 inference mode moves the flow of a trained network, by CPU emulation.

    python tools/bf16_accuracy.py -c CHECKPOINT.params [--hw 384x512] [--pairs 2] [--seed 0] [--max-disp 6]
                                  [--threads N] [--json FILE]

The checkpoint (a reference .params file, MaskFlownet-S or the cascade, told apart by its parameter names) comes from
the command line only; nothing in the repository reads one.

Runs the float reference graph oracle/network_ref.py (CPU; its C operators need the oracle library that
`__graft_entry__.build()` compiles) twice on the same image pairs:
    fp32  every convolution (3x3, stride-2, dilated, transposed) evaluated in float64, rounded once to fp32 -- the
          fp32-accurate mode, whose kernels err by ~2^-17 per product;
    bf16  the same with the bf16 mode's arithmetic: input and weight of every convolution rounded once to bf16 (nearest
          even), products and sums in float64; the outputs the mode stores as bf16 activations (the dense blocks
          conv{L}_0..4 and dc_conv1..6) rounded to bf16 after the LeakyReLU, as the kernel's epilogue stores them.
Correlation, the deformable warp, Upsample and the image warp are the oracle's fp32 operators in both runs, as they are
in both modes of the GPU path.  The convolutions are swapped in through the `tF` name network_ref calls them by, and
put back afterwards; the oracle itself is not modified.

The image pairs are synthetic with a known answer: a seeded smooth texture T (a sum of random sinusoids per channel)
and a seeded smooth flow f (random low-frequency sinusoids plus a random affine field, at most --max-disp pixels), with
im2 = T and im1(p) = T(p + f(p)) evaluated analytically, so that im1(p) = im2(p + f(p)) holds exactly and f is the
ground truth.  Prints, per precision, the mean end-point error against f at full resolution, and the mean and maximum
|flow_bf16 - flow_fp32| (per-pixel end-point distance), in pixels.  This is an emulation: the GPU kernels sum in a
different order, which changes results by far less than the bf16 rounding does.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import math
import os
import re
import sys
import time
import types

import numpy as np
import torch
import torch.nn.functional as tF

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import params as mparams  # noqa: E402
from oracle import cref, network_ref  # noqa: E402

STORED_BF16 = re.compile(r"(conv\d_[0-4]|dc_conv[1-6])\.weight$")   # outputs kept as bf16 activations in the bf16 mode


def _bf16(t: torch.Tensor) -> torch.Tensor:
    return t.to(torch.bfloat16).to(t.dtype)


@contextlib.contextmanager
def emulated_convolutions(precision: str, params: dict):
    """Replace network_ref's convolutions (its `tF` namespace) for the duration of the block.  precision "fp32": float64
    arithmetic; "bf16": bf16-rounded operands, float64 sums, bf16-stored outputs rounded after the activation."""
    by_ptr = {v.data_ptr(): k for k, v in params.items()}
    stored = {"pending": False}

    def operands(x, w):
        x, w = x.double(), w.double()
        if precision == "bf16":
            x, w = _bf16(x), _bf16(w)
        return x, w

    def conv2d(x, w, b=None, stride=1, padding=0, dilation=1):
        name = by_ptr.get(w.data_ptr(), "")
        xd, wd = operands(x, w)
        y = tF.conv2d(xd, wd, None if b is None else b.double(), stride, padding, dilation).float()
        stored["pending"] = precision == "bf16" and bool(STORED_BF16.search(name))
        return y

    def conv_transpose2d(x, w, b=None, stride=1, padding=0):
        xd, wd = operands(x, w)
        stored["pending"] = False
        return tF.conv_transpose2d(xd, wd, None if b is None else b.double(), stride, padding).float()

    def leaky_relu(y, slope):
        out = tF.leaky_relu(y, slope)
        if stored["pending"]:          # the activation of a convolution whose output the kernel stores as bf16
            out = _bf16(out)
        stored["pending"] = False
        return out

    shim = types.SimpleNamespace(conv2d=conv2d, conv_transpose2d=conv_transpose2d, leaky_relu=leaky_relu)
    saved = network_ref.tF
    network_ref.tF = shim
    try:
        yield
    finally:
        network_ref.tF = saved


def synthetic_pair(seed: int, H: int, W: int, max_disp: float):
    """(im1, im2) float32 (1,3,H,W) in [0,1] and the ground-truth flow (1,2,H,W), (y, x) in pixels: im1(p) = im2(p + f)."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)

    def texture(y, x):
        chans = []
        for _ in range(3):
            v = np.zeros_like(y)
            for _ in range(24):
                k = g.uniform(0.01, 0.12)                        # cycles per pixel: smooth but textured
                th, ph, a = g.uniform(0, 2 * np.pi), g.uniform(0, 2 * np.pi), g.uniform(0.2, 1.0)
                v = v + a * np.sin(2 * np.pi * k * (np.cos(th) * x + np.sin(th) * y) + ph)
            chans.append(v)
        t = np.stack(chans)
        return t

    # the flow: an affine field plus low-frequency sinusoids, scaled to max_disp
    f = []
    for _ in range(2):
        v = g.uniform(-1, 1) * (yy - H / 2) / H + g.uniform(-1, 1) * (xx - W / 2) / W + g.uniform(-0.5, 0.5)
        for _ in range(3):
            k = g.uniform(0.002, 0.01)
            th, ph = g.uniform(0, 2 * np.pi), g.uniform(0, 2 * np.pi)
            v = v + g.uniform(0.2, 0.6) * np.sin(2 * np.pi * k * (np.cos(th) * xx + np.sin(th) * yy) + ph)
        f.append(v)
    f = np.stack(f)
    f *= max_disp / np.abs(f).max()
    state = g.bit_generator.state                                # the same texture for both images
    t2 = texture(yy, xx)
    g.bit_generator.state = state
    t1 = texture(yy + f[0], xx + f[1])
    lo, hi = t2.min(), t2.max()
    im1 = ((t1 - lo) / (hi - lo)).clip(0, 1)
    im2 = ((t2 - lo) / (hi - lo)).clip(0, 1)
    as_t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))[None]  # noqa: E731
    return as_t(im1), as_t(im2), as_t(f)


def load_params(path: str):
    """name -> fp32 tensor under network_ref's names, and whether the checkpoint is the cascade (its head's parameters
    carry the `maskflownet_s` prefix)."""
    raw = mparams.read_params(path)
    cascade = any("maskflownet_s" in k for k in raw)
    return {mparams.gluon_to_module_name(k, cascade): torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32))
            for k, v in raw.items()}, cascade


def network_flow(params, cascade: bool, im1, im2, threads: int):
    """Full-resolution flow (1,2,H,W), (y, x) pixels: /255-free inputs in [0,1], centralise, forward, Upsample(4)."""
    mean = torch.cat([im1, im2], dim=2).mean(dim=(2, 3), keepdim=True)
    a, b = im1 - mean, im2 - mean
    if cascade:
        preds, _ = network_ref.maskflownet_forward(params, a, b, threads=threads)
    else:
        preds, _, _ = network_ref.maskflownet_s_forward(params, a, b, threads=threads)
    return torch.from_numpy(cref.upsample(preds[-1].numpy(), 4)).double()


def epe(a, b):
    return (a - b).square().sum(dim=1).sqrt()


def run(params, cascade, H, W, pairs, seed, max_disp, threads):
    res = {"fp32": [], "bf16": [], "delta_mean": [], "delta_max": []}
    for i in range(pairs):
        im1, im2, gt = synthetic_pair(seed + i, H, W, max_disp)
        flows = {}
        for prec in ("fp32", "bf16"):
            with emulated_convolutions(prec, params):
                flows[prec] = network_flow(params, cascade, im1, im2, threads)
            res[prec].append(float(epe(flows[prec], gt.double()).mean()))
        d = epe(flows["bf16"], flows["fp32"])
        res["delta_mean"].append(float(d.mean()))
        res["delta_max"].append(float(d.max()))
    return {"epe_fp32": float(np.mean(res["fp32"])), "epe_bf16": float(np.mean(res["bf16"])),
            "delta_mean": float(np.mean(res["delta_mean"])), "delta_max": float(np.max(res["delta_max"])),
            "per_pair": res}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("-c", "--checkpoint", required=True, help="a reference .params checkpoint (MaskFlownet-S or cascade)")
    ap.add_argument("--hw", default="384x512", help="image size HxW, multiples of 64")
    ap.add_argument("--pairs", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--max-disp", type=float, default=6.0, help="largest ground-truth displacement, pixels")
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1, help="threads of the C oracle's operators")
    ap.add_argument("--json", default="")
    a = ap.parse_args(argv)
    H, W = (int(s) for s in a.hw.lower().split("x"))
    if H % 64 or W % 64:
        ap.error("--hw must be multiples of 64 (the network's input grid)")
    params, cascade = load_params(a.checkpoint)
    t0 = time.perf_counter()
    r = run(params, cascade, H, W, a.pairs, a.seed, a.max_disp, a.threads)
    r.update(checkpoint=os.path.basename(a.checkpoint), network="MaskFlownet" if cascade else "MaskFlownet_S", hw=[H, W],
             pairs=a.pairs, seed=a.seed, max_disp=a.max_disp, seconds=round(time.perf_counter() - t0, 1),
             emulation="CPU: float64 convolutions, bf16-rounded operands / stored outputs in the bf16 run")
    print(f"{r['checkpoint']} ({r['network']}, {H}x{W}, {a.pairs} pairs, CPU emulation): mean EPE fp32 {r['epe_fp32']:.4f} px, "
          f"bf16 {r['epe_bf16']:.4f} px; |flow_bf16 - flow_fp32| mean {r['delta_mean']:.4f} px, max {r['delta_max']:.4f} px")
    if not math.isfinite(r["epe_bf16"]):
        sys.exit("non-finite flow")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(r, f, indent=1)
    return r


if __name__ == "__main__":
    main()
