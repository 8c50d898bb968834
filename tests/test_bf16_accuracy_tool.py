"""tools/bf16_accuracy.py on the CPU with random-init weights (no checkpoint is read): the synthetic pair carries its
ground-truth flow, the convolution swap is undone afterwards, the fp32 emulation is the oracle's forward to fp32
accuracy, and the bf16 emulation differs from it by bf16-sized amounts."""
import os
import sys

import torch

from maskflownet_b200 import network
from oracle import cref, network_ref

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import bf16_accuracy as acc  # noqa: E402


def test_synthetic_pair_satisfies_its_flow():
    im1, im2, f = acc.synthetic_pair(3, 64, 96, 4.0)
    assert im1.shape == im2.shape == (1, 3, 64, 96) and f.shape == (1, 2, 64, 96)
    assert 3.99 < float(f.abs().max()) <= 4.0 + 1e-6
    # im1(p) = im2(p + f(p)): bilinear sampling of im2 at p + f reproduces im1 away from the border, up to the
    # interpolation error of a smooth texture
    warped = torch.from_numpy(cref.reconstruction2d(im2.numpy(), f.numpy()))
    inner = (slice(None), slice(None), slice(8, -8), slice(8, -8))
    err = (warped - im1)[inner].abs()
    assert float(err.mean()) < 0.02 and float((torch.roll(im2, 5, 3) - im1)[inner].abs().mean()) > 0.05


def test_emulated_convolutions():
    torch.manual_seed(0)
    params = {k: v.detach().clone().contiguous() for k, v in network.MaskFlownetS().state_dict().items()}
    im1, im2, _ = acc.synthetic_pair(1, 64, 128, 3.0)
    saved = network_ref.tF
    plain = acc.network_flow(params, False, im1, im2, threads=1)
    flows = {}
    for prec in ("fp32", "bf16"):
        with acc.emulated_convolutions(prec, params):
            assert network_ref.tF is not saved
            flows[prec] = acc.network_flow(params, False, im1, im2, threads=1)
        assert network_ref.tF is saved
    scale = float(plain.abs().max())
    d32 = float((flows["fp32"] - plain).abs().max())
    d16 = float((flows["bf16"] - flows["fp32"]).abs().max())
    assert d32 <= 1e-4 * scale, (d32, scale)            # float64 sums vs the oracle's fp32 convolutions
    assert 1e-4 * scale < d16 <= 0.1 * scale, (d16, scale)   # operands with 8 significant bits
