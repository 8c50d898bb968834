"""Where the GPU time of one eager MaskFlownet-S forward goes, grouped by network part.

    python tools/step_profile.py [--batch 8] [--height 448] [--width 1024] [--precision fp32|bf16] [--json FILE]

Runs the forward of BASELINE configs[1] (batch 8, 1024x448, seeded inputs and weights) once under torch.profiler with
CUDA activities.  Every convolution call (ops.conv3x3_slices / ops.conv3x3_split) and every warp (ops.warp_mask) is
wrapped in a record_function range named after the layer that issued it; each kernel is attributed to the innermost
range around its launch (through the launch's correlation id in the trace) and summed into one of these groups:

    pyramid L1-L3     conv{1,2,3}{a,b,c} (both images in one batch)
    pyramid L4-L6     conv{4,5,6}{a,b,c}
    decoders L4-L6    the convolutions of the decoders whose input is at most 64 pixels wide: dense blocks, fused heads,
                      heads tail, upfeat, conv{L}f and the warp's convolution (levels 4-6, and upfeat3, whose input is
                      level 4)
    L2/L3             the same at levels 2 and 3, and the context network
    non-convolution   every other kernel: correlation, the warp's sampling, packing, copies, element-wise

Times are the sums of kernel durations (the profiler's), not wall time; the eager forward's wall time (CUDA events, no
profiler) is printed beside them.
"""
from __future__ import annotations

import argparse
import collections
import json
import os
import re
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import network, ops  # noqa: E402

GROUPS = ("pyramid L1-L3", "pyramid L4-L6", "decoders L4-L6", "L2/L3", "non-convolution")
CONV_KERNEL = re.compile(r"conv3x3")


def group_of(label: str, kernel: str) -> str:
    """label: 'layer|W' of the innermost range around the launch ('' outside every range)."""
    if not label or not CONV_KERNEL.search(kernel):
        return "non-convolution"
    layer, w = label.rsplit("|", 1)
    m = re.fullmatch(r"conv(\d)[abc]", layer)
    if m:
        return "pyramid L1-L3" if int(m.group(1)) <= 3 else "pyramid L4-L6"
    return "decoders L4-L6" if int(w) <= 64 else "L2/L3"


def attribute(trace_path: str):
    """[(kernel name, duration us, label)] from a chrome trace of torch.profiler."""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ranges = collections.defaultdict(list)   # tid -> [(ts, end, name)]
    launch = {}                              # correlation -> (tid, ts)
    kernels = []
    for e in ev:
        if e.get("ph") != "X":
            continue
        cat = e.get("cat", "")
        if cat == "user_annotation" and e["name"].startswith("mfn:"):
            ranges[e["tid"]].append((e["ts"], e["ts"] + e["dur"], e["name"][4:]))
        elif cat == "cuda_runtime" and "correlation" in e.get("args", {}):
            launch[e["args"]["correlation"]] = (e["tid"], e["ts"])
        elif cat == "kernel":
            kernels.append((e["name"], float(e["dur"]), e.get("args", {}).get("correlation")))
    out = []
    for name, dur, corr in kernels:
        label = ""
        if corr in launch:
            tid, ts = launch[corr]
            best = None
            for t0, t1, lab in ranges.get(tid, ()):
                if t0 <= ts <= t1 and (best is None or t0 >= best[0]):
                    best = (t0, lab)
            label = best[1] if best else ""
        out.append((name, dur, label))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=448)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--precision", choices=("fp32", "bf16"), default="fp32", help="the model's inference_precision")
    ap.add_argument("--json", default="", help="also write the groups and the per-label kernel times to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("step_profile.py times GPU kernels: no CUDA device")
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

    orig_slices, orig_split, orig_warp = ops.conv3x3_slices, ops.conv3x3_split, ops.warp_mask

    def slices(buf_in, *a, **k):
        with torch.profiler.record_function(f"mfn:{current['name']}|{buf_in.shape[-1]}"):
            return orig_slices(buf_in, *a, **k)

    def split(x, *a, **k):
        with torch.profiler.record_function(f"mfn:{current['name']}|{x.shape[-1]}"):
            return orig_split(x, *a, **k)

    def warp(feat, *a, **k):
        with torch.profiler.record_function(f"mfn:warp|{feat.shape[-1]}"):
            return orig_warp(feat, *a, **k)

    network._FlowNetBase._packed, network._FlowNetBase._packed_fn = packed, packed_fn
    ops.conv3x3_slices, ops.conv3x3_split, ops.warp_mask = slices, split, warp
    try:
        with torch.no_grad():
            for _ in range(3):
                network.predict_flow(model, a, b)            # warm-up: packing, kernel attributes
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            network.predict_flow(model, a, b)
            e1.record()
            torch.cuda.synchronize()
            wall = e0.elapsed_time(e1)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                    torch.profiler.ProfilerActivity.CUDA]) as prof:
                network.predict_flow(model, a, b)
                torch.cuda.synchronize()
    finally:
        network._FlowNetBase._packed, network._FlowNetBase._packed_fn = orig_packed, orig_packed_fn
        ops.conv3x3_slices, ops.conv3x3_split, ops.warp_mask = orig_slices, orig_split, orig_warp
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        rows = attribute(path)

    groups = collections.OrderedDict((gname, [0.0, 0]) for gname in GROUPS)
    per_label = collections.defaultdict(float)
    for name, dur, label in rows:
        gr = groups[group_of(label, name)]
        gr[0] += dur
        gr[1] += 1
        per_label[label or "(none)"] += dur
    total = sum(v[0] for v in groups.values())
    dev = torch.cuda.get_device_name()
    print(f"# {dev}; {args.precision}; batch {args.batch}, {args.width}x{args.height}; eager forward {wall:.3f} ms "
          f"(CUDA events, no profiler); {len(rows)} kernels, {total / 1e3:.3f} ms of kernel time")
    print(f"{'group':16s} {'kernels':>7s} {'ms':>8s} {'share':>6s}")
    for gname, (t, n) in groups.items():
        print(f"{gname:16s} {n:7d} {t / 1e3:8.3f} {t / total:6.1%}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": dev, "precision": args.precision, "batch": args.batch, "eager_forward_ms": wall,
                       "kernel_ms": total / 1e3,
                       "groups": {k: {"ms": v[0] / 1e3, "kernels": v[1]} for k, v in groups.items()},
                       "labels_ms": {k: v / 1e3 for k, v in sorted(per_label.items(), key=lambda kv: -kv[1])}},
                      f, indent=1)


if __name__ == "__main__":
    main()
