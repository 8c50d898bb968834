"""Every kernel launch of the benchmarked forwards against float64, at the benchmark's own shapes.

The shape of a launch decides which code runs: the split-K plan (small levels, and the short last round of a persistent
grid of one CTA per SM), the TMA box geometry of each dilation, the staged or register epilogue, the warp path.  Small
test shapes reach few of the combinations the benchmark runs, so this file runs the four benchmarked forwards once each
and checks every launch while it happens.  A recorder wraps the `ops` functions the graph calls; each wrapper runs the
original, synchronises, and compares that launch's output with a float64 reference of the same operation on the inputs
the kernel actually read (hi + lo of a split activation).  Every launch is judged on its own, so errors do not compound.
The references are plain torch in float64 on the GPU (cuDNN fp64 convolutions, oracle/torch_ref), one sample at a time.

Bound, per output element, with Q = sqrt(x^2 (*) w^2) (the scale of random rounding errors) and S = |x| (*) |w| + |b|:
    tensor-core launches (bf16 hi/lo split operands, fp32 accumulation)    |got - ref| <= 2^-12 Q + 2^-20 S
    exact-fp32 launches (SIMT warp, sampler, upsample)                      |got - ref| <= 2^-20 S
    plus, where the output is stored as a split activation (bf16 hi + lo), its rounding 2^-16 |ref| (split_storage_term).
The split's expected error is ~2^-17 Q; a bf16-only product errs by ~2^-9 Q and a dropped tap by ~Q / 3.  Where the
reference's pre-activation is below -bound the LeakyReLU scales the error by its slope, and so the bound.

Sampled operators read at positions computed in fp32.  The warp's reference computes its tap positions with the fp32
roundings of the tap-by-tap kernel and MXNet, fl((y - 1 + i) + fl(fl(f * scale) / stride)), from the up-sampled flow f
the kernel returned; the SIMT kernel rounds exactly so.  The warp through linearity samples the zero-corner operator
at the one position fl(y + d) moved by whole pixels and applies the MXNet-1.5 band correction at the per-tap positions;
where the two parts cancel (taps in the one-pixel bands) their rounding differences do not.  Its bound adds the position
deviation 2^-22 (|p| + |d| + 2) px per axis (p the pixel, d the displacement) times the slope of each part: twice the
zero-corner operator's plus the MXNet operator's.  The image warp rounds p + d after an fp32 Upsample(4); its bound adds
2^-20 (|p| + |d| + 1) px per axis times the reference's slope.  Slopes are one-sided differences, the steeper side.

The checker's sensitivity is asserted: on one real launch of each kind (fp32 NCHW, split in / split out, depth-to-space,
linear prefix, dilation >= 4) it must reject, by at least 3x, x and w rounded once to bf16 and one dropped tap.
test_checker_separates_kernel_arithmetic_from_near_misses checks the same on the CPU with the kernel's arithmetic
emulated.  Coverage is asserted too: the number of checked convolutions equals the graph's, each launch ran the kernel
variant its Cout selects, the cascade's level-2 split-K tail with split output ran, the TMA input ran at dilations
1, 2, 4, 8 and 16, and the cascade's level-6 warp ran through linearity at F = 196.

One line per launch is printed (pytest -s): op, layer, kernel, shape, dilation / stride, split-K workspace bytes, max
err / Q and max err / bound.  Not checked here: the transposed convolutions of the training graph (torch autograd).
"""
import time

import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import network

from launchcheck import fp64_references  # noqa: F401
from launchcheck.bounds import (CONTROL_MARGIN, EPS_Q, EPS_S, _expected_convs, activate, channel_slopes,
                                conv_near_misses, conv_terms, judge)
from launchcheck.inputs import _images_u8, _named_model, named_init
from launchcheck.recorders import Recorder


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound accepts the kernel's arithmetic and rejects its near misses
# ------------------------------------------------------------------------------------------------------------------
def test_checker_separates_kernel_arithmetic_from_near_misses():
    """The widest decoder layer (dc_conv1 at level 2: 579 -> 128), small image: the kernel's arithmetic (x and w split
    into bf16 hi + lo; hi*hi + hi*lo + lo*hi, each term accumulated in fp32) passes the bound, a bf16-only result and a
    dropped tap fail it by more than CONTROL_MARGIN."""
    g = torch.Generator().manual_seed(5)
    Cin, Cout, H, W = 579, 128, 10, 18
    a = torch.randn((1, Cin, H, W), generator=g)
    x = torch.where(a > 0, a, 0.1 * a)
    w = named_init("dc_conv1.weight", (Cout, Cin, 3, 3))
    b = named_init("dc_conv1.bias", (Cout,))

    def split(t):
        hi = t.bfloat16().float()
        return hi, (t - hi).bfloat16().float()
    (xh, xl), (wh, wl) = split(x), split(w)
    conv32 = lambda p, q: tF.conv2d(p, q, padding=1)  # noqa: E731
    kern = tF.leaky_relu(conv32(xh, wh) + conv32(xh, wl) + conv32(xl, wh) + b.view(1, -1, 1, 1), 0.1)

    pre, Q, S = conv_terms(x.double(), w.double(), b.double())
    bound = EPS_Q * Q + EPS_S * S
    sl = channel_slopes(Cout, 0.1)
    ratio, err_q = judge(kern, pre, sl, bound, Q)
    assert ratio <= 1.0 and err_q < 2.0 ** -14, (ratio, err_q)
    for name, alt in conv_near_misses(x.double(), w.double(), b.double()).items():
        r, _ = judge(activate(alt, sl), pre, sl, bound, Q)
        assert r >= CONTROL_MARGIN, (name, r)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the recorder
# ------------------------------------------------------------------------------------------------------------------
RUNS = {   # run: (model class, batch, H, W, image seed) -- bench.py's configs[1], [3], [4] (padded frame) and [2]
    "fwd": (network.MaskFlownetS, 8, 448, 1024, 21),
    "cascade": (network.MaskFlownet, 4, 448, 1024, 22),
    "odd": (network.MaskFlownetS, 4, 576, 960, 23),
    "train": (network.MaskFlownetS, 8, 384, 512, 24),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
@pytest.mark.usefixtures("fp64_references")
def test_every_launch_of_the_benchmarked_forward_against_float64(run, monkeypatch):
    cls, N, H, W, seed = RUNS[run]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    rec = Recorder(monkeypatch, run)         # before the model packs anything
    model = _named_model(cls)
    u1, u2 = _images_u8(seed=seed, n=N, h=H, w=W)
    if run == "train":
        model.train()
        a, b, _ = network.centralize(u1.float() / 255.0, u2.float() / 255.0)
        with torch.enable_grad():
            preds = model(a, b)[0]
        assert preds[-1].requires_grad
    else:
        model.eval()
        flow = network.predict_flow(model, u1, u2)
        assert flow.shape == (N, 2, H, W) and bool(torch.isfinite(flow).all())
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    rec.report()
    print(f"{run}: {len(rec.rows)} launches checked in {secs:.1f} s, peak {peak:.2f} GiB allocated")
    assert not rec.failures, "\n".join(rec.failures)

    # coverage: this run checked what the benchmark runs
    convs = [r for r in rec.rows if r["op"] in ("conv3x3_slices", "conv3x3_split")]
    assert len(convs) == _expected_convs(run), (len(convs), _expected_convs(run))
    print(f"{run}: kernel variants {sorted({r['kernel'] for r in convs})}")
    want_kinds = {"fp32", "dil>=4"} if run == "train" else set(Recorder.KINDS)
    assert set(rec.controls) == want_kinds, sorted(rec.controls)
    for tag, (name, rs) in rec.controls.items():
        assert min(rs.values()) >= CONTROL_MARGIN, (tag, name, rs)
    if run != "train":
        tma_dils = {r["dil"] for r in convs if r["op"] == "conv3x3_split"}
        assert {1, 2, 4, 8, 16} <= tma_dils, tma_dils
    if run == "cascade":
        assert any(r["split_out"] and r["ws"] > 0 and r["N"] == 4 and r["H"] == 112 for r in convs), \
            "no split-K launch with split output at level 2"
        assert any(r["op"] == "warp_mask" and r["kernel"] == "warp_lin_kernel" and r["Cout"] == 196 for r in rec.rows)
