"""Bidirectional flow with occlusion masks: one shared-pyramid forward against two one-way forwards, and the consistency
kernel alone.

    python tools/bidir_bench.py [--batch 8] [--hw 448x1024] [--rounds 5] [--steps 20] [--nets S,cascade]

bench.py's method: seeded uint8 pairs, random-init weights (seed 0), every step replayed from a CUDA graph, a 256 MiB L2
flush before every step, CUDA events around `steps` steps, `rounds` rounds.  The arms alternate inside each round, in one
process, so that clock and neighbour drift hit them alike.  Per network:
  a_bidirectional   one graph of network.predict_bidirectional: one pyramid pass for both directions, decoder at 2N,
                    one postprocess of 2N flows, one mfn_flow_consistency
  b_two_predicts    two graphs of network.predict, on (a,b) and on (b,a), then one ops.flow_consistency on their flows
  c_one_way         one graph of network.predict on (a,b), for scale
ms_per_step is the median over rounds; spread is (max - min) / median over rounds.
kernel: mfn_flow_consistency alone at N x 436 x 1024 (smooth consistent flows and noise), back to back from a CUDA graph,
against its byte bound: 2 N H W (8 + 8 + 1) B (the pixel's own flow, the four-corner gather of the other flow counted once,
the mask) over the 3.35 TB/s HBM3 data-sheet bandwidth of the H100 SXM.
Prints one JSON object with the card's name, power limit and SM clocks, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from maskflownet_b200 import network, ops  # noqa: E402

HBM_PEAK = 3.35e12
NETS = {"S": network.MaskFlownetS, "cascade": network.MaskFlownet}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def captured(fn, warmup=2):
    """fn() captured in a CUDA graph after warm-up calls on a side stream; returns (graph, outputs of the capture)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    return graph, out


def timed_ms(step, steps, flush):
    """ms per step over exactly `steps` steps, a 256 MiB L2 flush before each (inside the region), CUDA events."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        flush.zero_()
        step()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


@torch.no_grad()
def bench_net(cls, batch, H, W, rounds, steps, flush):
    torch.manual_seed(0)
    model = cls().cuda().eval()
    g = torch.Generator().manual_seed(100)
    a = torch.randint(0, 256, (batch, 3, H, W), dtype=torch.uint8, generator=g).cuda()
    b = torch.randint(0, 256, (batch, 3, H, W), dtype=torch.uint8, generator=g).cuda()
    g_bi, out_bi = captured(lambda: network.predict_bidirectional(model, a, b))
    g_ab, out_ab = captured(lambda: network.predict(model, a, b))
    g_ba, out_ba = captured(lambda: network.predict(model, b, a))

    def two_predicts():
        g_ab.replay()
        g_ba.replay()
        return ops.flow_consistency(out_ab[0], out_ba[0])

    arms = {"a_bidirectional": g_bi.replay, "b_two_predicts": two_predicts, "c_one_way": g_ab.replay}
    for fn in arms.values():   # warm every arm's shapes once more outside the timed region
        fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed_ms(fn, steps, flush))
    res = {}
    for k, ts in times.items():
        med = float(np.median(ts))
        res[k] = {"ms_per_step": round(med, 3), "spread": round((max(ts) - min(ts)) / med, 4),
                  "rounds_ms": [round(t, 3) for t in ts]}
    res["a_over_b"] = round(res["a_bidirectional"]["ms_per_step"] / res["b_two_predicts"]["ms_per_step"], 4)
    # both arms compute the same thing: report how far apart their flows and masks are
    g_bi.replay()
    occ_b = two_predicts()
    torch.cuda.synchronize()
    res["max_flow_diff_px"] = round(max(float((out_bi[0] - out_ab[0]).abs().max()),
                                        float((out_bi[1] - out_ba[0]).abs().max())), 6)
    res["mask_agreement"] = round(float(((out_bi[2] == occ_b[0]).float().mean() +
                                         (out_bi[3] == occ_b[1]).float().mean()) / 2), 6)
    res["occluded_share"] = round(float(out_bi[2].float().mean()), 4)
    del g_bi, g_ab, g_ba, model
    torch.cuda.empty_cache()
    return res


def kernel_time(fw, bw, iters=100, replays=5):
    graph, _ = captured(lambda: [ops.flow_consistency(fw, bw) for _ in range(iters)], warmup=1)
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        graph.replay()
    e1.record()
    e1.synchronize()
    t = e0.elapsed_time(e1) / 1e3 / (iters * replays)
    nbytes = 2 * (fw.numel() // 2) * (8 + 8 + 1)
    return {"us": round(t * 1e6, 2), "bytes": nbytes, "GB_s": round(nbytes / t / 1e9, 1),
            "share_of_hbm_peak": round(nbytes / t / HBM_PEAK, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--hw", default="448x1024")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--nets", default="S,cascade")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bidir_bench.py: no CUDA device")
    H, W = map(int, a.hw.split("x"))
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"gpu": gpu_info(), "batch": a.batch, "hw": [H, W], "rounds": a.rounds, "steps": a.steps, "nets": {}}
    for name in a.nets.split(","):
        res["nets"][name] = bench_net(NETS[name], a.batch, H, W, a.rounds, a.steps, flush)
    rng = np.random.default_rng(0)
    N, KH, KW = 8, 436, 1024
    y, x = np.mgrid[0:KH, 0:KW].astype(np.float32)
    rot = np.stack([-(y - KH / 2), x - KW / 2], -1) * 0.02
    smooth = np.broadcast_to(rot, (N, KH, KW, 2)) + rng.standard_normal((N, KH, KW, 2)).astype(np.float32) * 0.2
    noise = rng.standard_normal((N, KH, KW, 2)).astype(np.float32) * 10
    res["kernel"] = {}
    for fname, f in (("smooth", smooth), ("noise", noise)):
        fw = torch.from_numpy(np.ascontiguousarray(f, dtype=np.float32)).cuda()
        res["kernel"][fname] = kernel_time(fw, (-fw).contiguous())
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
