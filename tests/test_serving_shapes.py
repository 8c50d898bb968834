"""Every forward launch against float64 at the shapes a user's own frames reach, and the graph-replayed predictors
against the eager forward.

test_bench_shapes.py checks every launch at the four shapes bench.py times.  network.predict, VideoFlowPredictor and
tools/predict_new_data.py run other shapes -- one pair at a time, KITTI frames (375x1242, padded to 384x1280), HD video
(1080x1920, padded to 1088x1920), images down to 64x64 -- and there the dispatch differs:
  * plan_split (csrc/conv3x3_wgmma.cu) splits every tile at levels 3 and 4 of a single 448x1024 pair, and at level 2 of
    384x1280 and 1088x1920 only the tail rows of the one sample (n_lo = 0);
  * below 4 px ops.warp_mask leaves the through-linearity path: the 2x2 level 5 of a 64x64 pair runs warp_mma_kernel,
    the cascade's 1x1 level-6 warp (F = 196) the SIMT deform_fwd_kernel;
  * the 1x1 correlation has every displacement but the centre outside the image, and the dilation-16 context layer on
    a 16x16 level 2 has every off-centre tap outside: its TMA boxes lie wholly out of bounds.
test_split_plans_of_the_serving_shapes pins those plans on the CPU (mfn_conv3x3_workspace_bytes is host arithmetic).
test_every_launch_of_a_serving_forward_against_float64 runs five forwards through launchcheck's ServingRecorder,
with its bound and controls, and asserts that each run reached the path it is there for.  Controls added here, each to
be rejected by CONTROL_MARGIN: replicate padding instead of zero padding (the dilation-16 layer, the 1x1 correlation:
an out-of-bounds box that read the image), the last 16-channel chunk dropped on a split-every-tile launch (a lost
split-K part drops at least that), bf16-only operands and a dropped tap on the warp_mma_kernel launch.  The kitti and hd
runs also compare ops.preprocess (with its resize) and ops.postprocess with oracle/prepost_ref on the same inputs.

The graph paths that give bench.py its numbers, FlowPredictor (a CUDA-graph replay) and PipelinedFlowPredictor (pinned
host buffers, copy streams, staging slots), are compared with the eager forward bit for bit at the benchmark's shapes,
under torch.use_deterministic_algorithms(True): that selects the deterministic preprocessing mean (otherwise the
forward's one run-to-run difference) and fills every torch.empty with NaN, so a kernel that reads a buffer before
writing it shows up as a non-finite or different flow.

Not checked here: the backward at these shapes, frames larger than 1088x1920.
"""
import time

import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import _lib, network

from launchcheck import fp64_references  # noqa: F401
from launchcheck.bounds import (CONTROL_MARGIN, EPS_Q, EPS_S, _expected_convs, channel_slopes, conv_terms, judge,
                                split_storage_term)
from launchcheck.inputs import _deterministic, _images_u8, _named_model, _same, named_init
from launchcheck.recorders import Recorder, ServingRecorder, _cover_tiny, _cover_tiny_cascade


# ------------------------------------------------------------------------------------------------------------------
# CPU: the split-K plans the serving runs are there to reach
# ------------------------------------------------------------------------------------------------------------------
def test_split_plans_of_the_serving_shapes():
    """plan_split (csrc/conv3x3_wgmma.cu) for named layers of the serving runs, N = 1: 132 SMs, tiles of 2 rows x 128 px.
    Every tile split when 2 x tiles <= 132: k = min(132 // tiles, chunks // 3, 8) parts, ws = 4 k N Cout OH OW bytes.
    Tail split (a short last round, Cout > 64, >= 16 chunks): the tiles past the last full round of 132, widened to whole
    tile rows, in min(132 // tail, chunks // 2) parts; ws = 4 k Cout rh OW bytes over the rows [OH - rh, OH)."""
    wb = _lib.lib().mfn_conv3x3_workspace_bytes
    # tiny (64x64): every decoder level splits every tile, the 1x1 level 6 included
    assert wb(1, 81, 1, 1, 128, 1, 1) == 2 * 128 * 4                  # conv6_0: 6 chunks -> 2 parts
    assert wb(1, 497, 1, 1, 36, 1, 1) == 8 * 36 * 4                   # conv6_4 + heads
    assert wb(1, 483, 2, 2, 96, 1, 1) == 8 * 96 * 2 * 2 * 4           # conv5_2
    assert wb(1, 451, 4, 4, 96, 1, 1) == 8 * 96 * 4 * 4 * 4           # conv4_2
    assert wb(1, 419, 8, 8, 96, 1, 1) == 8 * 96 * 8 * 8 * 4           # conv3_2
    assert wb(1, 387, 16, 16, 96, 1, 1) == 8 * 96 * 16 * 16 * 4       # conv2_2: 8 tiles
    assert wb(1, 96, 16, 16, 64, 1, 16) == 2 * 64 * 16 * 16 * 4       # dc_conv5, dilation 16: 6 chunks -> 2 parts
    assert wb(1, 32, 16, 16, 2, 1, 1) == 0                             # dc_conv7: 2 chunks, nothing to split
    # single (448x1024): levels 3 (28 tiles) and 4 (14 tiles) split every tile, which batch 8 never does
    assert wb(1, 419, 56, 128, 96, 1, 1) == 4 * 96 * 56 * 128 * 4      # conv3_2: 132 // 28 = 4
    assert wb(1, 451, 28, 64, 96, 1, 1) == 8 * 96 * 28 * 64 * 4        # conv4_2: min(132 // 14, 29 // 3, 8)
    assert wb(1, 195, 28, 64, 128, 1, 1) == 4 * 128 * 28 * 64 * 4      # conv4_0: 13 chunks -> 4
    assert wb(1, 579, 112, 256, 128, 1, 1) == 0                        # level 2: 112 tiles, one short round
    # kitti (384x1280): level 2 is 96x320, 3 tiles per row (2.5 tiles of pixels), 144 tiles = 132 + 12: the last 12 are
    # tile rows 44..47 = rows 88..95 of the only sample, in 132 // 12 = 11 parts
    assert wb(1, 387, 96, 320, 96, 1, 1) == 11 * 96 * 8 * 320 * 4      # conv2_2
    assert wb(1, 579, 96, 320, 128, 1, 1) == 11 * 128 * 8 * 320 * 4    # dc_conv1
    assert wb(1, 259, 96, 320, 128, 1, 1) == 8 * 128 * 8 * 320 * 4     # conv2_1: 17 chunks -> 8
    assert wb(1, 483, 96, 320, 64, 1, 1) == 0                          # conv2_3: Cout 64 does not gain
    # hd (1088x1920): level 2 is 272x480, 4 tiles per row (3.75), 544 tiles = 4 x 132 + 16: tile rows 132..135 = rows
    # 264..271 in 132 // 16 = 8 parts; level 3 (136x240, 136 tiles = 132 + 4): rows 132..135 in 19 // 2 = 9 parts
    assert wb(1, 579, 272, 480, 128, 1, 1) == 8 * 128 * 8 * 480 * 4    # dc_conv1
    assert wb(1, 387, 272, 480, 96, 1, 1) == 8 * 96 * 8 * 480 * 4      # conv2_2
    assert wb(1, 291, 136, 240, 128, 1, 1) == 9 * 128 * 4 * 240 * 4    # conv3_1
    # level 6 is 17x30 (odd height, rows of 30 px): 9 tiles, every tile split
    assert wb(1, 337, 17, 30, 96, 1, 1) == 7 * 96 * 17 * 30 * 4        # conv6_2: 21 chunks -> 7


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound holds for a bias-dominated output stored as a split activation
# ------------------------------------------------------------------------------------------------------------------
def test_split_output_storage_term_covers_a_bias_dominated_output():
    """conv6_0 on a 1x1 level 6: the md=4 correlation input is zero but for the centre displacement, so Q = |w x| is
    tiny and the output is nearly the bias.  The kernel's arithmetic (hi/lo split operands, fp32 sums, LeakyReLU) with
    an fp32 output passes 2^-12 Q + 2^-20 S; stored as a split activation (bf16 hi + lo of the fp32 value) it needs the
    storage term 2^-16 |ref| of split_storage_term, which it then passes."""
    w = named_init("conv6_0.weight", (128, 81, 3, 3))
    b = named_init("conv6_0.bias", (128,))
    sl = channel_slopes(128, 0.1)

    def split(t):
        hi = t.bfloat16().float()
        return hi, (t - hi).bfloat16().float()
    worst = {"fp32": 0.0, "split, no term": 0.0, "split": 0.0}
    for v in (0.0123, -0.0071, 0.031, 0.0042):
        x = torch.zeros((1, 81, 1, 1))
        x[0, 40] = v
        (xh, xl), (wh, wl) = split(x), split(w)
        conv32 = lambda p, q: tF.conv2d(p, q, padding=1)  # noqa: E731
        out = tF.leaky_relu(conv32(xh, wh) + conv32(xh, wl) + conv32(xl, wh) + b.view(1, -1, 1, 1), 0.1)
        oh, ol = split(out)
        pre, Q, S = conv_terms(x.double(), w.double(), b.double())
        bound = EPS_Q * Q + EPS_S * S
        worst["fp32"] = max(worst["fp32"], judge(out, pre, sl, bound, Q)[0])
        worst["split, no term"] = max(worst["split, no term"], judge(oh.double() + ol.double(), pre, sl, bound, Q)[0])
        worst["split"] = max(worst["split"], judge(oh.double() + ol.double(), pre, sl,
                                                   bound + split_storage_term(pre, 0), Q)[0])
    assert worst["fp32"] <= 1.0 and worst["split"] <= 1.0 and worst["split, no term"] > 1.0, worst


# ------------------------------------------------------------------------------------------------------------------
# GPU: the five serving forwards
# ------------------------------------------------------------------------------------------------------------------
def _cover_single(rec, convs):
    for h in (56, 28):      # levels 3 and 4
        split = [r for r in convs if r["op"] == "conv3x3_split" and r["H"] == h and r["ws"] > 0]
        assert len(split) >= 5 and all(r["split_all"] and r["N"] == 1 for r in split), (h, split)
    assert "chunk" in rec.extra


def _tail_rows_8(r):
    """A tail split of rows [OH - 8, OH) of the only sample: ws = 4 k Cout 8 OW."""
    return r["ws"] > 0 and not r["split_all"] and r["ws"] % (4 * r["Cout"] * 8 * r["W"]) == 0


def _cover_prepost(rec, net_hw):
    pre = [r for r in rec.rows if r["op"] == "preprocess"]
    post = [r for r in rec.rows if r["op"] == "postprocess"]
    assert len(pre) == 1 and pre[0]["name"] == f"-> {net_hw[0]}x{net_hw[1]}" and len(post) == 2


def _cover_kitti(rec, convs):
    lvl2 = [r for r in convs if r["op"] == "conv3x3_split" and (r["H"], r["W"]) == (96, 320)]
    assert lvl2 and sum(_tail_rows_8(r) for r in lvl2) >= 3, lvl2    # conv2_1, conv2_2, dc_conv1: rows 88..95
    _cover_prepost(rec, (384, 1280))


def _cover_hd(rec, convs):
    # an odd-height level 6 with 30-px rows, fp32 outputs included (rows of 30 floats are not 16-byte aligned, which by
    # conv3x3_wgmma_launch's `staged` condition sends them to the register epilogue; which epilogue ran is not
    # observable from here, only that these launches ran and were checked)
    assert any((r["H"], r["W"]) == (17, 30) and not r["split_out"] for r in convs)
    lvl2 = [r for r in convs if r["op"] == "conv3x3_split" and (r["H"], r["W"]) == (272, 480)]
    assert lvl2 and sum(_tail_rows_8(r) for r in lvl2) >= 3, lvl2    # rows 264..271
    _cover_prepost(rec, (1088, 1920))


SERVING = {   # run: (model class, batch, input H, W, image seed, through network.predict, coverage)
    "tiny": (network.MaskFlownetS, 1, 64, 64, 31, False, _cover_tiny),
    "tiny_cascade": (network.MaskFlownet, 1, 64, 64, 32, False, _cover_tiny_cascade),
    "single": (network.MaskFlownetS, 1, 448, 1024, 33, False, _cover_single),
    "kitti": (network.MaskFlownetS, 1, 375, 1242, 34, True, _cover_kitti),
    "hd": (network.MaskFlownetS, 1, 1080, 1920, 35, True, _cover_hd),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(SERVING))
@pytest.mark.usefixtures("fp64_references")
def test_every_launch_of_a_serving_forward_against_float64(run, monkeypatch):
    cls, N, H, W, seed, via_predict, cover = SERVING[run]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    rec = ServingRecorder(monkeypatch, run)         # before the model packs anything
    model = _named_model(cls).eval()
    u1, u2 = _images_u8(seed=seed, n=N, h=H, w=W)
    if via_predict:
        flow, occ = network.predict(model, u1, u2)
        assert flow.shape == (N, H, W, 2) and occ.shape == (N, H, W, 1)
    else:
        flow = network.predict_flow(model, u1, u2)
        assert flow.shape == (N, 2, H, W)
    assert bool(torch.isfinite(flow).all())
    torch.cuda.synchronize()
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    rec.report()
    print(f"{run}: {len(rec.rows)} launches checked in {secs:.1f} s, peak {peak:.2f} GiB allocated")
    assert not rec.failures, "\n".join(rec.failures)

    convs = [r for r in rec.rows if r["op"] in ("conv3x3_slices", "conv3x3_split")]
    assert len(convs) == _expected_convs("cascade" if cls is network.MaskFlownet else "fwd"), len(convs)
    assert set(Recorder.KINDS) <= set(rec.controls), sorted(rec.controls)
    for tag, (name, rs) in rec.controls.items():
        assert min(rs.values()) >= CONTROL_MARGIN, (tag, name, rs)
    for tag, (name, r) in rec.extra.items():
        assert r >= CONTROL_MARGIN, (tag, name, r)
    cover(rec, convs)


# ------------------------------------------------------------------------------------------------------------------
# GPU: the serving paths against eager, bit for bit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("arch,N,conv,deform", [("S", 8, "conv5_1", "deform4"), ("cascade", 4, "conv4_1", "deform3")])
def test_flow_predictor_graph_equals_eager_at_the_benchmark_shape(arch, N, conv, deform):
    """FlowPredictor (bench.py's judged value) replays the eager forward bit for bit: on two pairs, on the first again
    after the second, and after an in-place weight change followed by invalidate()."""
    model = _named_model(network.MaskFlownetS if arch == "S" else network.MaskFlownet).eval()
    p1 = _images_u8(seed=41, n=N, h=448, w=1024)
    p2 = _images_u8(seed=42, n=N, h=448, w=1024)
    with _deterministic():
        e1 = network.predict_flow(model, *p1).clone()
        _same(network.predict_flow(model, *p1), e1, f"{arch}: eager twice")
        e2 = network.predict_flow(model, *p2).clone()
        pred = network.FlowPredictor(model)
        _same(pred(*p1), e1, f"{arch}: graph, pair 1")
        _same(pred(*p2), e2, f"{arch}: graph, pair 2")
        _same(pred(*p1), e1, f"{arch}: graph, pair 1 after pair 2")
        with torch.no_grad():
            getattr(model, conv).weight.mul_(1.25)
            getattr(model, deform).weight.mul_(0.75)
        pred.invalidate()
        e3 = network.predict_flow(model, *p1).clone()
        assert not torch.equal(e3, e1), "the weight change did not change the flow"
        _same(pred(*p1), e3, f"{arch}: graph after the weight change")
        torch.cuda.synchronize()


@pytest.mark.gpu
def test_pipelined_predictor_equals_eager_at_the_benchmark_shape():
    """PipelinedFlowPredictor(depth=2): five distinct pinned pairs enqueued into five pinned outputs without a
    synchronisation in between; the last output is complete once the event its infer() returned has completed, and every
    output equals the eager flow after synchronize()."""
    model = _named_model(network.MaskFlownetS).eval()
    with _deterministic():
        pairs, refs = [], []
        for i in range(5):
            a, b = _images_u8(seed=50 + i, n=8, h=448, w=1024)
            refs.append(network.predict_flow(model, a, b).cpu())
            pairs.append((a.cpu().pin_memory(), b.cpu().pin_memory()))
        outs = [torch.full((8, 2, 448, 1024), float("nan")).pin_memory() for _ in range(5)]
        pipe = network.PipelinedFlowPredictor(model, depth=2)
        torch.cuda.synchronize()
        evs = [pipe.infer(a, b, o) for (a, b), o in zip(pairs, outs)]
        evs[-1].synchronize()
        _same(outs[-1], refs[-1], "pipelined: last output after its event")
        pipe.synchronize()
        for i in range(5):
            _same(outs[i], refs[i], f"pipelined: request {i}")


@pytest.mark.gpu
def test_pipelined_predictor_gives_each_shape_its_own_slots():
    """A batch-8 request at 448x1024, a batch-2 request at 64x128 (a 1x2 level 6), then batch 8 again: each equals the
    eager flow."""
    model = _named_model(network.MaskFlownetS).eval()
    reqs = [_images_u8(seed=60, n=8, h=448, w=1024), _images_u8(seed=61, n=2, h=64, w=128),
            _images_u8(seed=62, n=8, h=448, w=1024)]
    with _deterministic():
        refs = [network.predict_flow(model, a, b).cpu() for a, b in reqs]
        host = [(a.cpu().pin_memory(), b.cpu().pin_memory()) for a, b in reqs]
        outs = [torch.full(tuple(r.shape), float("nan")).pin_memory() for r in refs]
        pipe = network.PipelinedFlowPredictor(model, depth=2)
        for (a, b), o in zip(host, outs):
            pipe.infer(a, b, o)
        pipe.synchronize()
        for i, (o, r) in enumerate(zip(outs, refs)):
            _same(o, r, f"pipelined: request {i} {tuple(r.shape)}")
