"""Inputs of the launch checks: models with the golden fixture's named initialisation, seeded images and clips, and the
deterministic-algorithms switch with the bit-equality assertion of the graph-replay tests."""
import contextlib
import os
import sys

import numpy as np
import torch

from maskflownet_b200 import network

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "golden"))
from make_golden import gluon_to_module_name, named_init, seeded_images  # noqa: E402,F401

FLOW_HEAD_SCALE = 1.0 / 16       # keeps random flow heads' flows small: tests/test_unsup_step_launches.py says why


def _named_model(cls):
    m = cls()
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(named_init(k.replace("MaskFlownet_S.", "") if cls is network.MaskFlownetS else k, p.shape))
    return m.cuda()


def _images_u8(seed, n, h, w):
    out = []
    for t in seeded_images(seed=seed, n=n, h=h, w=w):
        lo, hi = t.amin(), t.amax()
        out.append(((t - lo) / (hi - lo) * 255).round().to(torch.uint8).contiguous().cuda())
    return out


def _scaled_model(cls):
    model = _named_model(cls).eval()
    with torch.no_grad():
        for k, p in model.named_parameters():
            if "pred_flow" in k or "dc_conv7" in k:
                p.mul_(FLOW_HEAD_SCALE)
    return model


def _clip(seed, T, H, W):
    """T uint8 frames (T,3,H,W) on the device: one seeded image moving by (2, -3) px per frame."""
    base = _images_u8(seed=seed, n=1, h=H, w=W)[0][0]
    return torch.stack([torch.roll(base, shifts=(2 * t, -3 * t), dims=(1, 2)) for t in range(T)]).contiguous()


@contextlib.contextmanager
def _deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _same(got, ref, what):
    assert bool(torch.isfinite(ref).all()), f"{what}: the eager flow is not finite"
    d = (got.float() - ref.float()).abs()
    assert torch.equal(got, ref), f"{what}: max |diff| {float(d.nan_to_num(float('inf')).max()):.3g} at " \
                                  f"{np.unravel_index(int(d.nan_to_num(float('inf')).argmax()), tuple(d.shape))}"
