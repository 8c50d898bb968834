"""One convolution run with the TMA-staged input and with the per-thread loads, and its float64 check."""
import numpy as np
import torch

from maskflownet_b200 import _lib, ops


DEV = "cuda"


def feat(rng, shape):
    a = rng.standard_normal(shape).astype(np.float32)
    return np.where(a > 0, a, 0.1 * a).astype(np.float32)


def reference(x, w, b, dil=1, stride=1, slope=0.1):
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, stride=stride,
                                     padding=dil, dilation=dil)
    ref = ref + torch.from_numpy(b).double().view(1, -1, 1, 1)
    return torch.nn.functional.leaky_relu(ref, slope).numpy()


def run_both(x_full, c0, Cin, w, b, stride=1, dil=1, bf16=False, grid_cap=0, shift=0):
    """conv3x3_slices of channels [c0, c0 + Cin) of x_full into channels [2, 2 + Cout) of a NaN-filled buffer, with the
    TMA-staged input (knob 1) and with the per-thread loads (knob 0); returns (output slice, kernel name with knob 1,
    kernel name with knob 0) after checking the two outputs are bit-identical, ran the same variant, and nothing outside
    the slice was written.
    shift > 0 places the input `shift` floats past the start of its allocation."""
    N, _, H, W = x_full.shape
    Cout = w.shape[0]
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    flat = torch.zeros(x_full.size + shift, device=DEV)
    flat[shift:] = torch.from_numpy(x_full).to(DEV).flatten()
    xg = flat[shift:].view(x_full.shape)
    pk = ops.conv3x3_pack(torch.from_numpy(w).to(DEV))
    bg = torch.from_numpy(b).to(DEV)
    res = {}
    try:
        _lib.set_tuning("conv_grid_cap", grid_cap)
        for knob in (0, 1):
            _lib.set_tuning("conv_tma_in", knob)
            out = torch.full((N, Cout + 3, OH, OW), float("nan"), device=DEV)
            ops.conv3x3_slices(xg, c0, Cin, pk, bg, out, 2, Cout, 0.1, dilation=dil, stride=stride, bf16=bf16)
            torch.cuda.synchronize()
            res[knob] = (out.cpu(), _lib.last_kernel())
    finally:
        _lib.set_tuning("conv_tma_in", 1)
        _lib.set_tuning("conv_grid_cap", 0)
    (o0, k0), (o1, k1) = res[0], res[1]
    assert torch.equal(o0.isnan(), o1.isnan()) and torch.equal(torch.nan_to_num(o0), torch.nan_to_num(o1)), (k1, k0)
    assert o1[:, :2].isnan().all() and o1[:, 2 + Cout:].isnan().all(), k1
    assert k0 == k1, (k0, k1)
    return o1[:, 2:2 + Cout].numpy(), k1, k0


def check(got, x, w, b, stride=1, dil=1, bf16=False):
    ref = reference(x, w, b, dil, stride)
    tol = 3e-2 if bf16 else 1e-4
    err = float(np.abs(got - ref).max())
    assert err <= tol * max(1.0, float(np.abs(ref).max())), err


def weights(rng, Cout, Cin):
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    return w, (rng.standard_normal(Cout) * 0.1).astype(np.float32)
