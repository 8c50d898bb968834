"""Split activations (ops.SplitAct, include/maskflow_b200.h: mfn_split_pack / mfn_conv3x3_forward_split): the packed
values are the bf16 hi/lo split of the fp32 values, and a convolution that reads its input from a split buffer (tensor
copies) and / or writes its output into one gives bit for bit the result of the fp32 path (conv3x3_slices) -- for partial
and whole input chunks, linear prefixes, dilations 1, 2, 4, 8 and 16, staged and register epilogues, the split-K plans
(small images, and a short last round reduced into split output) and capped persistent grids.  Whole networks: the flows
equal those of the fp32 dense block exactly."""
import pytest
import torch

from maskflownet_b200 import _lib, network, ops

pytestmark = pytest.mark.gpu
DEV = "cuda"


def leaky(shape, g):
    a = torch.randn(shape, generator=g).to(DEV)
    return torch.where(a > 0, a, 0.1 * a)


def test_pack_round_trip():
    g = torch.Generator().manual_seed(0)
    x = leaky((2, 35, 5, 33), g) * 1e3
    act = ops.SplitAct(2, 51, 5, 33, DEV)
    act.buf.fill_(0xFF)
    act.pack(x, 16)
    hi, lo = act.hi_lo()
    want_hi = x.bfloat16().float()
    assert torch.equal(hi[:, 16:], want_hi)
    assert torch.equal(lo[:, 16:], (x - want_hi).bfloat16().float())
    # the pad channels of the slice (51 .. 63) are zeros in both planes
    raw = act.buf.view(2, 2, 8, 5, 33, 16)
    assert int(raw[:, :, 6, :, :, 6:].abs().sum()) == 0 and int(raw[:, :, 7].abs().sum()) == 0


CASES = [   # (N, Cin, H, W, Cout, linear prefix, dilation[, grid cap that makes the last round short])
    (2, 131, 6, 256, 32, 0, 1),     # partial last chunk, staged fp32 epilogue
    (2, 547, 4, 256, 34, 2, 1),     # conv2_4 + heads
    (2, 547, 5, 130, 36, 4, 1),     # conv3_4 + heads (padded prefix), register epilogue
    (2, 131, 6, 256, 96, 0, 2),
    (1, 128, 5, 130, 128, 0, 16),
    (2, 259, 4, 130, 128, 0, 1),
    (8, 675, 14, 32, 64, 0, 1),     # level 5: split-K over the input chunks
    (8, 547, 7, 16, 34, 2, 1),      # level 6 conv6_4 + heads: split-K with a linear prefix and split output (reduce kernel)
    (1, 128, 40, 130, 128, 0, 16),  # dilation 16 with in-bounds rows for every tap
    (1, 128, 10, 130, 128, 0, 4),   # dc_conv3: dilation 4, rows partly in bounds
    (2, 128, 18, 130, 96, 0, 8),    # dc_conv4: dilation 8, rows partly in bounds
    # short last round on a 12-CTA grid (28 tiles = 2 x 12 + 4): the last sample's tail rows split over 3 parts and
    # reduced into the split output (y_lo > 0, n_lo > 0)
    (2, 259, 14, 130, 96, 0, 1, 12),
]


@pytest.mark.parametrize("cap", [0, 1, 3])
@pytest.mark.parametrize("case", CASES)
def test_split_conv_is_bit_identical(case, cap):
    N, Cin, H, W, Cout, lp, dil, *last_round_cap = case
    if cap and N * Cin * H > 20000:
        pytest.skip("grid caps: the small shapes suffice")
    if last_round_cap:
        if cap:
            pytest.skip("the case brings its own grid cap")
        cap = last_round_cap[0]
    g = torch.Generator().manual_seed(Cin + Cout)
    x = leaky((N, Cin + 16, H, W), g)          # the convolution reads channels [16, 16 + Cin)
    w = torch.randn((Cout, Cin, 3, 3), generator=g).to(DEV) / (3 * Cin ** 0.5)
    b = torch.randn(Cout, generator=g).to(DEV)
    packed = ops.conv3x3_pack(w)
    _lib.set_tuning("conv_grid_cap", cap)
    try:
        if last_round_cap:    # the tail of the last sample only: a proper part of the output
            assert 0 < _lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, 1, dil) < 4 * N * Cout * H * W
        ref = torch.empty((N, Cout, H, W), device=DEV)
        ops.conv3x3_slices(x, 16, Cin, packed, b, ref, 0, Cout, 0.1, dil, linear_prefix=lp)
        xs = ops.SplitAct(N, Cin + 16, H, W, DEV)
        xs.pack(x, 0)
        # split in, fp32 out
        y = torch.empty_like(ref)
        ops.conv3x3_split(xs, 16, Cin, packed, b, Cout, 0.1, dil, out=y, linear_prefix=lp)
        assert torch.equal(y, ref)
        # split in, split out (channels 32.. of the output buffer), prefix to fp32
        want = ops.SplitAct(N, 32 + Cout - lp, H, W, DEV)
        want.buf.zero_()
        want.pack(ref[:, lp:].contiguous(), 32)
        got = ops.SplitAct(N, 32 + Cout - lp, H, W, DEV)
        got.buf.zero_()
        pre = torch.empty((N, lp, H, W), device=DEV) if lp else None
        ops.conv3x3_split(xs, 16, Cin, packed, b, Cout, 0.1, dil, out=pre, out_split=got, out_c0=32, linear_prefix=lp)
        assert torch.equal(got.buf, want.buf)
        if lp:
            assert torch.equal(pre, ref[:, :lp])
    finally:
        _lib.set_tuning("conv_grid_cap", 0)


def test_split_conv_rejects_bad_slices():
    xs = ops.SplitAct(1, 64, 4, 8, DEV)
    packed = ops.conv3x3_pack(torch.zeros((16, 20, 3, 3), device=DEV))
    y = torch.empty((1, 16, 4, 8), device=DEV)
    with pytest.raises(_lib.MaskflowError, match="multiple of 16"):   # would read channels 36..47 as pad
        ops.conv3x3_split(xs, 16, 20, packed, None, 16, out=y)
    with pytest.raises(_lib.MaskflowError, match="overlap"):
        ops.conv3x3_split(xs, 16, 48, ops.conv3x3_pack(torch.zeros((16, 48, 3, 3), device=DEV)), None, 16, out_split=xs,
                          out_c0=48)
    with pytest.raises(_lib.MaskflowError, match="multiple of 16"):   # the pack would zero channels 21..31
        xs.pack(torch.zeros((1, 5, 4, 8), device=DEV), 16)


def test_split_depth_to_space_is_bit_identical():
    g = torch.Generator().manual_seed(7)
    N, Cin, H, W, F = 2, 611, 6, 128, 16
    x = leaky((N, Cin, H, W), g)
    w = torch.randn((Cin, F, 4, 4), generator=g).to(DEV) / 40
    b = torch.randn(F, generator=g).to(DEV)
    packed = ops.conv_transpose4x4_pack(w)
    ref = torch.empty((N, F, 2 * H, 2 * W), device=DEV)
    ops.conv3x3_slices(x, 0, Cin, packed, b, ref, 0, 4 * F, 0.1, depth_to_space=True)
    xs = ops.SplitAct(N, Cin, H, W, DEV)
    xs.pack(x, 0)
    y = torch.empty_like(ref)
    ops.conv3x3_split(xs, 0, Cin, packed, b, 4 * F, 0.1, out=y, depth_to_space=True)
    assert torch.equal(y, ref)


def _fp32_dense(self, lvl, x):
    """The fp32 dense block the split one replaced (same launches, fp32 concat buffer), as the reference."""
    N, Cb, H, W = x.shape
    front = sum(network.DECODER_CH)
    buf = torch.empty((N, front + Cb, H, W), device=x.device)
    buf[:, front:] = x
    off = front
    for i, oc in enumerate(network.DECODER_CH):
        conv = getattr(self, f"conv{lvl}_{i}")
        ops.conv3x3_slices(buf, off, buf.shape[1] - off, self._packed(f"conv{lvl}_{i}"), conv.bias, buf, off - oc, oc,
                           network.SLOPE)
        off -= oc
    act = ops.SplitAct(N, buf.shape[1], H, W, x.device)
    act.pack(buf, 0)
    return network._Slab(act, None, 0)


@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet])
def test_network_flows_equal_fp32_dense_block(cls, monkeypatch):
    torch.manual_seed(0)
    model = cls().to(DEV).eval()
    g = torch.Generator().manual_seed(1)
    a, b = torch.rand((2, 3, 128, 256), generator=g).to(DEV), torch.rand((2, 3, 128, 256), generator=g).to(DEV)
    with torch.no_grad():
        model.fuse_heads = False
        if cls is network.MaskFlownet:
            model.MaskFlownet_S.fuse_heads = False
        got = model(a, b)[0]
        monkeypatch.setattr(network._FlowNetBase, "_dense_split", _fp32_dense)
        want = model(a, b)[0]
    for p, q in zip(got, want):
        assert torch.equal(p, q)
