"""Every training-step launch against float64 at the reference's own dataset crops, with its robust loss.

test_bench_shapes_backward.py checks every forward and backward launch of the benchmarked training steps (384x512 and
576x960, a mask of ones, the L2 loss).  The reference trains elsewhere too (main.py, network/config/*.yaml):
  * FlyingChairs 384x512 cropped to 320x448, batch 8: levels 5x7 .. 80x112;
  * KITTI 370x1224 cropped to 320x896, batch 4, the robust loss q = 0.4 and a sparse validity mask: levels 5x14 .. 80x224;
  * Sintel / Things3D 436x1024 cropped to 384x768, batch 4, q = 0.4: levels 6x12 .. 96x192.
The loss sees the mask after the geometry augmentation: fractional, and for KITTI sparse.  This file builds each step the
way PipelineFlownet._train_batch does -- uint8 frames and a flow label at the dataset's size, augment.geometry_augment
with fixed draws, ColorAugmentation with the reference's arguments for the dataset, network.centralize, the model in train
mode, losses.multiscale_epe(eps=1e-8, q) and its backward -- and checks every launch while it happens with the recorders
Recorder (forward) and BackwardRecorder (backward) of launchcheck.recorders, bounds and controls included.

The KITTI runs also place exact zeros: after the forward the label of a patch is set to ops.upsample(preds[-1], 4), which
the loss kernel's own up-sampling reproduces bit for bit (asserted), so there d = 0 at scale 4, s = eps and the q-gradient's
sign is 0.  That is what the sign(0) = +1 control needs.  The cascade's run trains end to end (head included), so the image
warp's flow gradient -- the only path from the cascade's loss into the head's flow2 -- is checked too.
"""
import time

import pytest
import torch

from maskflownet_b200 import augment, losses, network

from launchcheck import fp64_references  # noqa: F401
from launchcheck.bounds import CONTROL_MARGIN
from launchcheck.inputs import _images_u8, _named_model
from launchcheck.recorders import BackwardRecorder, Recorder

EPS = 1e-8
# The q-gradient's bound is vacuous at an element where the box of the kernel's fp32 d leaves it no tighter than the
# gradient's own size (pos >= S): there the sign is open because s_lo reached eps.  On an H100 the q runs had no such
# element at any scale (0 of 288 .. 147456).  That the box term dominates the rounding term (pos > gamma_L S) is common
# and harmless at the fine scales, where L is small: 60 - 99.7 % of the x4 elements, with err / bound <= 0.12.
# 1e-3 of a launch's elements (about 150 at x4) leaves room for a chance near-zero d while a vacuous region fails.
VACUOUS_MAX = 1e-3

DATASETS = {   # dataset: (orig, target, GeometryAugmentation, ColorAugmentation arguments) of the reference's main.py
    "chairs": ((384, 512), (320, 448),
               dict(angle_range=(-17, 17), zoom_range=(0.5, 1 / 0.9), aspect_range=(0.9, 1 / 0.9), translation_range=0.1,
                    relative_angle=0.25, relative_scale=(0.96, 1 / 0.96), relative_translation=0.25),
               dict(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4), noise_range=(0, 0.04),
                    saturation=0.5, hue=0.5)),
    "kitti": ((370, 1224), (320, 896),
              dict(angle_range=(-5, 5), zoom_range=(1 / 1.25, 1 / 0.95), aspect_range=(0.95, 1 / 0.95),
                   translation_range=0.05, relative_angle=0.25, relative_scale=(0.98, 1 / 0.98), relative_translation=0.25),
              dict(contrast_range=(-0.2, 0.4), brightness_sigma=0.05, channel_range=(0.9, 1.2), noise_range=(0, 0.02),
                   saturation=0.25, hue=0.1, gamma_range=(-0.5, 0.5))),
    "sintel": ((436, 1024), (384, 768),
               dict(angle_range=(-17, 17), zoom_range=(1 / 1.5, 1 / 0.9), aspect_range=(0.9, 1 / 0.9),
                    translation_range=0.1, relative_angle=0.25, relative_scale=(0.96, 1 / 0.96), relative_translation=0.25),
               dict(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4), noise_range=(0, 0),
                    saturation=0.5, hue=0.5)),
}

RUNS = {   # run: (dataset, model class, batch per GPU, q, deterministic, seed)
    "chairs": ("chairs", network.MaskFlownetS, 8, None, False, 41),
    "kitti": ("kitti", network.MaskFlownetS, 4, 0.4, False, 42),
    "kitti-det": ("kitti", network.MaskFlownetS, 4, 0.4, True, 42),
    "sintel": ("sintel", network.MaskFlownetS, 4, 0.4, False, 43),
    "sintel-cascade": ("sintel", network.MaskFlownet, 2, 0.4, False, 44),
}
PATCH = (slice(200, 264), slice(400, 528))     # the KITTI runs' exact-zero patch of the 320x896 crop


def _frames(dataset, N, seed):
    """uint8 frames, a float flow label in (x, y) order and a uint8 mask at the dataset's original size.  KITTI: a
    LiDAR-like validity mask -- the top third invalid, about a third of the rest valid at random -- and the label zero
    where invalid; otherwise the broadcast mask of ones PipelineFlownet uses when there is none."""
    (H, W), _, _, _ = DATASETS[dataset]
    u1, u2 = _images_u8(seed=seed, n=N, h=H, w=W)
    g = torch.Generator().manual_seed(seed)
    label = torch.randn(N, 2, H, W, generator=g) * 3
    if dataset == "kitti":
        valid = torch.rand(N, 1, H, W, generator=g) < 0.35
        valid[:, :, :H // 3] = False
        label = label * valid
        mask = valid.to(torch.uint8) * 255
    else:
        mask = torch.full((N, 1, 1, 1), 255, dtype=torch.uint8)
    return u1, u2, label.cuda(), mask.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
@pytest.mark.usefixtures("fp64_references")
def test_every_launch_of_a_dataset_training_step_against_float64(run, monkeypatch):
    dataset, cls, N, q, det, seed = RUNS[run]
    orig, target, geo_args, col_args = DATASETS[dataset]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fwd = Recorder(monkeypatch, run)
    bwd = BackwardRecorder(monkeypatch, run)
    model = _named_model(cls).train()
    u1, u2, label, mask = _frames(dataset, N, seed)
    geo = augment.GeometryAugmentation(target_shape=target, orig_shape=orig, batch_size=N, seed=seed, **geo_args)
    col = augment.ColorAugmentation(batch_size=N, shape=target, seed=seed + 1, **col_args)
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(det, warn_only=True)
    zero = None
    try:
        with torch.no_grad():
            i1, i2, flow, mask = geo(u1, u2, label, mask)
            i1, i2 = col(i1, i2)
            a, b, _ = network.centralize(i1, i2)
            flow = flow.flip(1).contiguous()            # the network's (y, x) order (pipeline.py:106)
        preds = model(a, b)[0]
        if dataset == "kitti":
            with torch.no_grad():
                up = fwd.orig["upsample"](preds[-1].detach(), 4)
                flow[:, :, PATCH[0], PATCH[1]] = up[:, :, PATCH[0], PATCH[1]]
            zero = torch.zeros_like(mask, dtype=torch.bool)
            zero[:, :, PATCH[0], PATCH[1]] = True
            bwd.exact_zero = (4, zero)
        losses.multiscale_epe(flow, mask, preds, eps=EPS, q=q).sum().backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    fwd.report()
    bwd.report()
    print(f"{run}: {len(fwd.rows)} forward and {len(bwd.rows)} backward checks in {secs:.1f} s, peak {peak:.2f} GiB")

    # the exact zeros are exact: with the mask on the patch only, the x4 q-gradient is 0 everywhere (sign(0) = 0), which
    # holds only if the loss kernel's up-sampled prediction equals ops.upsample's bit for bit at every patch pixel
    if zero is not None:
        p4 = preds[-1].detach().clone().requires_grad_()
        patch_mask = (mask * zero).contiguous()
        assert float(patch_mask.sum()) > 100
        losses.multiscale_epe(flow, patch_mask, [p4], scales=(4,), weights=(1.0,), eps=EPS, q=q).sum().backward()
        assert int((p4.grad != 0).sum()) == 0, "ops.upsample and the loss's upsample2_at differ on the patch"

    assert not fwd.failures, "\n".join(fwd.failures)
    assert not bwd.failures, "\n".join(bwd.failures)

    # the mask reached the loss fractional (and, for KITTI, sparse)
    if dataset == "kitti":
        assert bool(((mask > 0) & (mask < 1)).any()) and float((mask == 0).float().mean()) > 0.3

    # coverage: the graph's launch counts
    corr = [r for r in bwd.rows if r["op"] == "corr_bwd"]
    warps = bwd.calls.count("mfn_warp_mask_backward") + bwd.calls.count("mfn_warp_mask_backward_det")
    ups = [r for r in bwd.rows if r["op"] == "upsample_bwd"]
    convs_fwd = [r for r in fwd.rows if r["op"] == "conv3x3_slices"]
    convs_bwd = [r for r in bwd.rows if r["op"] == "conv_bwd"]
    cascade = cls is network.MaskFlownet
    assert len(corr) == 5 + (10 if cascade else 0), len(corr)
    assert warps == 4 + (5 if cascade else 0), warps
    assert len(ups) == 8 + (7 if cascade else 0), len(ups)
    epe_b = [r for r in bwd.rows if r["op"] == "epe_bwd"]
    epe_f = [r for r in bwd.rows if r["op"] == "epe_fwd"]
    assert len(epe_b) == 5 and len(epe_f) == 1
    assert all(r["name"].endswith("q=0.4") for r in epe_b + epe_f) == (q is not None)
    assert len(convs_bwd) == len(convs_fwd), (len(convs_bwd), len(convs_fwd))
    if not cascade:
        assert len(convs_fwd) == 2 * 18 + 5 * 5 + 9 + 4 + 7
    iw = bwd.calls.count("mfn_image_warp_concat_backward") + bwd.calls.count("mfn_image_warp_concat_backward_det")
    assert iw == (1 if cascade else 0), iw
    if cascade:
        assert any(r["op"] == "image_warp_bwd" and r["name"] == "g_flow_up" for r in bwd.rows)
    if det:
        assert bwd.calls.count("mfn_warp_mask_backward_det") == 4
        atomic = {"mfn_warp_mask_backward", "mfn_deformable_conv_backward", "mfn_bilinear_sampler_backward",
                  "mfn_image_warp_concat_backward"}
        assert not atomic & set(bwd.calls), sorted(atomic & set(bwd.calls))

    # the q-gradient's bound is informative almost everywhere
    if q is not None:
        worst = max(n_vac / n for _, _, n_vac, n in bwd.epe_vacuous)
        assert worst <= VACUOUS_MAX, bwd.epe_vacuous

    # sensitivity: every control fails the bound by CONTROL_MARGIN on its launch
    want = {"corr md=4", "corr leaky", "upsample x2", "warp", "epe x64", "conv wiring"} | ({"corr md=2", "image warp"} if cascade else set())
    if q is not None:
        want |= {"epe L2 form"}
    if dataset == "kitti":
        want |= {"epe mask rounded", "epe sign(0) = +1"}
    assert want <= set(bwd.controls), sorted(bwd.controls)
    for kind, lst in bwd.controls.items():
        for entry in lst:
            assert min(entry[-1].values()) >= CONTROL_MARGIN, (kind, entry)
    if q is not None:
        assert len(bwd.controls["epe L2 form"]) == 2                 # forward and backward
    if dataset == "kitti":
        assert len(bwd.controls["epe mask rounded"]) == 2
