"""Where the time of the 3x3 / transposed convolutions goes, set against what the H100 can do.

    python tools/conv_bound.py [--batch 8] [--height 448] [--width 1024] [--reps 5] [--levels 2,3] [--json FILE]
                               [--precision fp32|bf16]

Runs one eager MaskFlownet-S forward (BASELINE configs[1]: batch 8, 1024x448, seeded inputs and weights) and records every
convolution launch (ops.conv3x3_slices / ops.conv3x3_split) with the layer that issued it.  Each recorded launch is then replayed on its own,
bracketed by CUDA events (median of --reps), in seven variants of the profiling knob `conv_dbg` of the wgmma kernel:

    full      the real kernel
    -load     producers skip their global loads (they still convert and hand over every stage)
    -input    producers skip loads, conversion and shared-memory stores (they only hand over every stage): what a free
              input path would cost
    -wload    the weight loader issues no bulk copies (it still hands over every weight stage)
    -feed     neither the input nor the weight stages are delivered (-input and -wload together): what the kernel would
              take if nothing had to reach shared memory
    -store    no epilogue stores
    -mma      no tensor-core MMAs (the barrier protocol is unchanged)

The variants give invalid results; replays only time, and the forward that recorded the calls ran before any of them.
Per launch the table prints the shape, the time, and two lower bounds:

    mma    the MMA slots the kernel issues (128-pixel x 2-row tiles, 64-pixel ones where the output is at most 64 pixels
           wide and at stride 2, padded input / output channels, three or two bf16
           products per fp32 product, whole rounds of one work item per SM) at the 989 TFLOP/s dense-bf16 data-sheet rate
    hbm    input + output + packed weights once over the 3.35 TB/s data-sheet bandwidth

and `frac` = max(mma, hbm) / time.  --precision bf16 runs the forward in the opt-in bf16 mode (inference_precision):
its launches issue one bf16 product per fp32 product, so the mma bound counts one (and the hbm bound reads bf16
activations at 2 bytes per channel-pixel).  The six deltas (time minus the time without a phase) show what each phase adds to
the critical path.  Both rates are for a 700 W part; a card with a lower power limit runs slower clocks.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import _lib, network, ops  # noqa: E402

PEAK_FLOPS, PEAK_BW, SMS = 989e12, 3.35e12, 132
R = 2   # rows per tile (csrc/conv3x3_wgmma.cu)


def tile_width(ow: int, stride: int) -> int:
    """Pixels per tile row (um::tile_width): one 64-pixel MMA block per row where the output is at most 64 wide, and at
    stride 2 (the TMA-staged input's tiles)."""
    return 64 if ow <= 64 or stride == 2 else 128


MODES = (("full", 0), ("-load", 2), ("-input", 16), ("-wload", 32), ("-feed", 48), ("-store", 4), ("-mma", 8))
DELTAS = ("-load", "-input", "-wload", "-feed", "-store", "-mma")


def cout_pad(cin: int, cout: int) -> int:
    """Output-channel padding of the wgmma kernel, read back from the size of its weight image (the mma.sync image in
    front of it pads to 32 / 64 / 96 / 128 and stops at 128 channels; csrc/conv3x3.cu)."""
    sync = ((cin + 31) // 32) * 9 * 2 * (-(-cout // 32) * 32) * 64 if cout <= 128 else 0
    return (int(_lib.lib().mfn_conv3x3_packed_bytes(cin, cout)) - sync) // (((cin + 15) // 16) * 9 * 64)


def mma_columns(cout_p: int, terms: int = 3) -> int:
    """Accumulator columns the MMAs of one 64-pixel block issue per tap and 16-channel chunk: three products over CoutP,
    or -- folded narrow layers -- hi x [hi; lo] over 2 CoutP plus lo x hi over CoutP; terms = 1 (bf16 mode): hi x hi over
    CoutP."""
    if cout_p > 128:
        return 2 * terms * 128
    return terms * cout_p


def bounds(c, terms=3):
    N, Cin, H, W, Cout, stride, dil = c["N"], c["Cin"], c["H"], c["W"], c["Cout"], c["stride"], c["dil"]
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    MT = tile_width(OW, stride)
    tiles = N * ((OW + MT - 1) // MT) * ((OH + R - 1) // R)
    chunks = (Cin + 15) // 16
    cp = cout_pad(Cin, Cout)
    k = 1
    if c["ws_bytes"]:   # split-K over chunks (levels 5-6): the plan cuts every tile into k parts
        k = max(1, c["ws_bytes"] // (4 * N * Cout * OH * OW))
    ns = 2 if cp > 128 else 1
    items = tiles * k * ns
    rounds = -(-items // SMS)
    per_item_flop = 2 * (R * MT) * 16 * mma_columns(cp, terms) // ns * 9 * (-(-chunks // k))
    mma = rounds * per_item_flop / (PEAK_FLOPS / SMS)
    useful = terms * 2 * N * OH * OW * Cout * Cin * 9 / PEAK_FLOPS
    Fo = Cout // 4 if c["d2s"] else Cout
    out_px = N * OH * OW * (4 if c["d2s"] else 1)
    ib = 2 if terms == 1 and "fn" in c else 4                                         # a bf16 activation in
    ob = 2 if terms == 1 and "fn" in c and c["args"][9] is not None else 4            # a bf16 activation out
    nbytes = ib * N * Cin * H * W + ob * Fo * out_px + int(_lib.lib().mfn_conv3x3_packed_bytes(Cin, Cout))
    return mma, nbytes / PEAK_BW, useful


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=448)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--levels", default="", help="comma-separated levels to list per layer (default: all)")
    ap.add_argument("--json", default="", help="also write the rows as JSON to this file")
    ap.add_argument("--precision", choices=("fp32", "bf16"), default="fp32", help="the model's inference_precision")
    args = ap.parse_args()
    terms = 1 if args.precision == "bf16" else 3
    if not torch.cuda.is_available():
        sys.exit("conv_bound.py times GPU kernels: no CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    model = network.MaskFlownetS().cuda().eval()
    model.inference_precision = args.precision
    g = torch.Generator().manual_seed(0)
    a = torch.randint(0, 256, (args.batch, 3, args.height, args.width), dtype=torch.uint8, generator=g).cuda()
    b = torch.randint(0, 256, (args.batch, 3, args.height, args.width), dtype=torch.uint8, generator=g).cuda()

    # the layer that issued a launch: the packed weight it was just handed (_packed / _packed_fn run right before the call)
    current = {"name": "?"}
    orig_packed, orig_packed_fn = network._FlowNetBase._packed, network._FlowNetBase._packed_fn

    def packed(self, name):
        current["name"] = name
        return orig_packed(self, name)

    def packed_fn(self, key, params, build):
        current["name"] = key
        return orig_packed_fn(self, key, params, build)

    calls, recording = [], {"on": False}
    orig_slices = ops.conv3x3_slices

    def slices(buf_in, c_in0, Cin, packed_w, bias, buf_out, c_out0, Cout, leaky_slope=0.1, dilation=1, stride=1,
               depth_to_space=False, linear_prefix=0, bf16=False):
        orig_slices(buf_in, c_in0, Cin, packed_w, bias, buf_out, c_out0, Cout, leaky_slope, dilation, stride, depth_to_space,
                    linear_prefix, bf16)
        if recording["on"]:
            N, _, H, W = buf_in.shape
            calls.append({"layer": current["name"], "N": N, "Cin": Cin, "H": H, "W": W, "Cout": Cout, "stride": stride,
                          "dil": dilation, "d2s": depth_to_space, "lin": linear_prefix,
                          "ws_bytes": int(_lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, stride, dilation)),
                          "args": (buf_in, c_in0, Cin, packed_w, bias, buf_out, c_out0, Cout, leaky_slope, dilation, stride,
                                   depth_to_space, linear_prefix, bf16)})

    orig_split = ops.conv3x3_split

    def split(x, c_in0, Cin, packed_w, bias, Cout, leaky_slope=0.1, dilation=1, out=None, out_split=None, out_c0=0,
              depth_to_space=False, linear_prefix=0, bf16=False):
        args = (x, c_in0, Cin, packed_w, bias, Cout, leaky_slope, dilation, out, out_split, out_c0, depth_to_space,
                linear_prefix, bf16)
        orig_split(*args)
        if recording["on"]:
            N, _, H, W = x.shape
            calls.append({"layer": current["name"], "N": N, "Cin": Cin, "H": H, "W": W, "Cout": Cout, "stride": 1,
                          "dil": dilation, "d2s": depth_to_space, "lin": linear_prefix,
                          "ws_bytes": int(_lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, 1, dilation)),
                          "fn": orig_split, "args": args})

    network._FlowNetBase._packed, network._FlowNetBase._packed_fn = packed, packed_fn
    ops.conv3x3_slices = slices
    ops.conv3x3_split = split
    with torch.no_grad():
        for _ in range(2):
            network.predict_flow(model, a, b)            # warm-up: packing, kernel attributes
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        recording["on"] = True
        e0.record()
        network.predict_flow(model, a, b)
        e1.record()
        recording["on"] = False
    ops.conv3x3_slices, ops.conv3x3_split = orig_slices, orig_split
    torch.cuda.synchronize()
    step = e0.elapsed_time(e1)

    def time_call(c):
        ts = []
        for _ in range(args.reps + 1):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            c.get("fn", orig_slices)(*c["args"])
            t1.record()
            ts.append((t0, t1))
        torch.cuda.synchronize()
        v = sorted(x.elapsed_time(y) for x, y in ts[1:])
        return v[len(v) // 2]

    try:
        for mode, dbg in MODES:
            _lib.set_tuning("conv_dbg", dbg)
            with torch.no_grad():
                for c in calls:
                    c[mode] = time_call(c)
    finally:
        _lib.set_tuning("conv_dbg", 0)

    dev = torch.cuda.get_device_name()
    print(f"# {dev}; {args.precision}; eager forward {step:.3f} ms; {len(calls)} convolution launches; "
          f"times in us (median of {args.reps}); bounds at 989 TFLOP/s bf16 and 3.35 TB/s, {terms} product(s) per MAC")
    want = {int(x) for x in args.levels.split(",") if x.strip()}
    hdr = (f"{'layer':16s} {'N':>2s} {'Cin':>4s} {'Cout':>4s} {'H':>4s} {'W':>5s} s d {'time':>8s} {'mma':>8s} {'hbm':>7s} "
           f"{'frac':>5s} " + " ".join(f"{k[1:]:>7s}" for k in DELTAS))
    print(hdr)
    per_level = collections.OrderedDict()
    NV = 4 + len(DELTAS)   # time, mma, hbm, useful, then the deltas
    rows = []
    for c in calls:
        mma, hbm, useful = bounds(c, terms)
        t = c["full"] * 1e-3
        m = re.search(r"\d", c["layer"])
        lvl = 2 if c["layer"].startswith("dc_conv") else (int(m.group()) if m else 0)
        kind = "pyramid" if re.fullmatch(r"conv\d[abc]", c["layer"]) else "decoder"
        grp = f"{kind} L{lvl}"
        d = {k: c["full"] - c[k] for k in DELTAS}
        row = {k: v for k, v in c.items() if k not in ("args", "fn")}
        row.update(level=lvl, group=grp, mma_us=mma * 1e6, hbm_us=hbm * 1e6, useful_us=useful * 1e6,
                   frac=max(mma, hbm) / t)
        rows.append(row)
        agg = per_level.setdefault(grp, [0.0] * NV + [0])
        for i, v in enumerate((c["full"], mma * 1e3, hbm * 1e3, useful * 1e3) + tuple(d[k] for k in DELTAS)):
            agg[i] += v
        agg[NV] += 1
        if want and lvl not in want:
            continue
        print(f"{c['layer']:16s} {c['N']:2d} {c['Cin']:4d} {c['Cout']:4d} {c['H']:4d} {c['W']:5d} {c['stride']} "
              f"{c['dil']:<2d}{c['full'] * 1e3:7.0f} {mma * 1e6:8.0f} {hbm * 1e6:7.0f} {max(mma, hbm) / t:5.2f} "
              + " ".join(f"{d[k] * 1e3:7.0f}" for k in DELTAS))
    print(f"\n{'group':12s} {'calls':>5s} {'time':>8s} {'mma':>8s} {'useful':>8s} {'hbm':>7s} {'frac':>5s} "
          + " ".join(f"{k[1:]:>7s}" for k in DELTAS) + "   (us; frac = mma bound / time)")
    tot = [0.0] * NV + [0]
    for grp, v in sorted(per_level.items(), key=lambda kv: -kv[1][0]):
        tot = [x + y for x, y in zip(tot, v)]
        print(f"{grp:12s} {v[NV]:5d} {v[0] * 1e3:8.0f} {v[1] * 1e3:8.0f} {v[3] * 1e3:8.0f} {v[2] * 1e3:7.0f} "
              f"{v[1] / v[0]:5.2f} " + " ".join(f"{x * 1e3:7.0f}" for x in v[4:NV]))
    print(f"{'all':12s} {tot[NV]:5d} {tot[0] * 1e3:8.0f} {tot[1] * 1e3:8.0f} {tot[3] * 1e3:8.0f} {tot[2] * 1e3:7.0f} "
          f"{tot[1] / tot[0]:5.2f} " + " ".join(f"{x * 1e3:7.0f}" for x in tot[4:NV]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": dev, "precision": args.precision, "eager_forward_ms": step, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
