"""The wgmma convolution's output widths and epilogues: output channels are padded to the next multiple of 16 (48, 80 and
112 included; narrow layers fold the hi / lo weight images into one operand), and whole tiles of plain NCHW output whose
rows are 16-byte aligned leave through shared-memory staging rows and bulk copies, while other outputs (unaligned
rows, depth-to-space, split-K parts) store from registers.  Every case is checked against a float64 convolution."""
import numpy as np
import pytest
import torch

from maskflownet_b200 import _lib, ops

DEV = "cuda"


def feat(rng, shape):
    a = rng.standard_normal(shape).astype(np.float32)
    return np.where(a > 0, a, 0.1 * a).astype(np.float32)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def reference(x, w, b, dil, d2s, lin):
    """float64 LeakyReLU(conv3x3 + bias) with the linear prefix and the depth-to-space layout of conv3x3_slices."""
    N, _, H, W = x.shape
    Cout = w.shape[0]
    F = Cout // 4 if d2s else Cout
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, padding=dil,
                                     dilation=dil)
    if d2s:      # conv channel (2 py + px) * F + f -> out[f][2y + py][2x + px]
        ref = ref.reshape(N, 2, 2, F, H, W).permute(0, 3, 4, 1, 5, 2).reshape(N, F, 2 * H, 2 * W)
    ref = ref + torch.from_numpy(b).double().view(1, F, 1, 1)
    act = torch.nn.functional.leaky_relu(ref, 0.1)
    if lin:
        act[:, :lin] = ref[:, :lin]
    return act.float().numpy()


def run_slices(x, w, b, dil, d2s, lin):
    """conv3x3_slices into channels [2, 2 + F) of a NaN-filled wider buffer; returns (written slice, buffer, kernel)."""
    N, Cin, H, W = x.shape
    Cout = w.shape[0]
    F = Cout // 4 if d2s else Cout
    out = torch.full((N, F + 3, (2 if d2s else 1) * H, (2 if d2s else 1) * W), float("nan"), device=DEV)
    ops.conv3x3_slices(cu(x), 0, Cin, ops.conv3x3_pack(cu(w)), cu(b), out, 2, Cout, 0.1, dilation=dil,
                       depth_to_space=d2s, linear_prefix=lin)
    kern = _lib.last_kernel()
    return out[:, 2:2 + F].cpu().numpy(), out, kern


def check(got, out, ref, F, kern):
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max())), kern
    assert torch.isnan(out[:, :2]).all() and torch.isnan(out[:, 2 + F:]).all(), kern   # nothing outside the slice


@pytest.mark.gpu
@pytest.mark.parametrize("Cout", [33, 35, 48, 72, 100])
@pytest.mark.parametrize("dil", [1, 2, 16])
@pytest.mark.parametrize("W", [136, 130])   # 136: rows 16-byte aligned (staged epilogue); 130: register epilogue
def test_padded_widths_match_float64(Cout, dil, W):
    rng = np.random.default_rng(61 + Cout + dil)
    N, Cin, H = 2, 70, 9
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    for lin in (0, 3):
        got, out, kern = run_slices(x, w, b, dil, False, lin)
        assert f"CoutP={(Cout + 15) // 16 * 16}" in kern, kern
        check(got, out, reference(x, w, b, dil, False, lin), Cout, kern)


@pytest.mark.gpu
@pytest.mark.parametrize("Cout", [48, 72, 100])
def test_padded_widths_depth_to_space(Cout):
    rng = np.random.default_rng(67 + Cout)
    N, Cin, H, W = 2, 40, 7, 132
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout // 4) * 0.1).astype(np.float32)
    got, out, kern = run_slices(x, w, b, 1, True, 0)
    check(got, out, reference(x, w, b, 1, True, 0), Cout // 4, kern)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [1, 3])
@pytest.mark.parametrize("Cout,W", [(35, 200), (100, 152), (128, 256), (48, 150)])
def test_persistent_grid_with_staged_epilogue(cap, Cout, W):
    """With the grid capped every CTA walks many tiles: the staging rows are reused while earlier bulk copies may still be
    reading them, and the rings wrap.  W = 200: the right-hand tile is partial (72 pixels); W = 150: register epilogue."""
    rng = np.random.default_rng(71 + cap + Cout)
    N, Cin, H = 2, 50, 13
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    _lib.set_tuning("conv_grid_cap", cap)
    try:
        got, out, kern = run_slices(x, w, b, 1, False, 2)
    finally:
        _lib.set_tuning("conv_grid_cap", 0)
    check(got, out, reference(x, w, b, 1, False, 2), Cout, kern)


@pytest.mark.gpu
def test_fused_head_layer_runs_the_48_wide_variant():
    """conv{L}_4 + heads of MaskFlownet-S (32 + 3 outputs) pads to 48 output channels, not 64."""
    rng = np.random.default_rng(73)
    N, Cin, H, W = 1, 67, 6, 64
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((35, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(35) * 0.1).astype(np.float32)
    got, out, kern = run_slices(x, w, b, 1, False, 3)
    assert kern == "conv3x3_wgmma_kernel<CoutP=48,fold>", kern
    check(got, out, reference(x, w, b, 1, False, 3), 35, kern)


@pytest.mark.parametrize("Cout,CoutP", [(2, 16), (16, 16), (33, 48), (35, 48), (64, 64), (72, 80), (100, 112), (128, 128),
                                        (196, 256)])
def test_packed_image_pads_to_multiples_of_16(Cout, CoutP):
    """Host arithmetic (no GPU): the wgmma weight image behind the mma.sync one holds CoutP padded rows per tap."""
    Cin = 70
    sync = ((Cin + 31) // 32) * 9 * 2 * (-(-Cout // 32) * 32) * 64 if Cout <= 128 else 0
    assert _lib.lib().mfn_conv3x3_packed_bytes(Cin, Cout) == sync + ((Cin + 15) // 16) * 9 * 64 * CoutP
