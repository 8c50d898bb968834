"""The wgmma convolution's 64-pixel tile rows (csrc/conv3x3_wgmma.cu, um::tile_width): outputs at most 64 pixels wide run
tiles of 2 rows x 64 pixels -- one m64 MMA block per output row instead of two, the second of which would lie wholly
right of the image.  The per-output arithmetic (products, chunk and tap order) is the 128-pixel tile's, so every
variant is compared bit for bit with the same launch on 128-pixel tiles (tuning knob conv_narrow = 0) and against a
float64 convolution, at widths 1, 16, 17, 30, 32 and 64: the fp32 input path (dilations 1 and 2, linear prefix,
depth-to-space, stride 2), the split input read by tensor copies (dilations 1, 2 and 4), split output, the linear-prefix
heads, split-K, a capped grid, and the bf16 mode."""
import numpy as np
import pytest
import torch

from maskflownet_b200 import _lib, ops

DEV = "cuda"
WIDTHS = [1, 16, 17, 30, 32, 64]


def feat(rng, shape):
    a = rng.standard_normal(shape).astype(np.float32)
    return np.where(a > 0, a, 0.1 * a).astype(np.float32)


def weights(rng, Cout, Cin, nb=None):
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(nb or Cout) * 0.1).astype(np.float32)
    return w, b


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def reference(x, w, b, dil=1, stride=1, d2s=False, lin=0, slope=0.1):
    """float64 LeakyReLU(conv3x3 + bias), the first `lin` channels linear, optionally depth-to-space."""
    N, _, H, W = x.shape
    Cout = w.shape[0]
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, stride=stride,
                                     padding=dil, dilation=dil)
    if d2s:      # conv channel (2 py + px) * F + f -> out[f][2y + py][2x + px]
        F = Cout // 4
        ref = ref.reshape(N, 2, 2, F, H, W).permute(0, 3, 4, 1, 5, 2).reshape(N, F, 2 * H, 2 * W)
    ref = ref + torch.from_numpy(b).double().view(1, -1, 1, 1)
    act = torch.nn.functional.leaky_relu(ref, slope)
    if lin:
        act[:, :lin] = ref[:, :lin]
    return act.numpy()


def both(run):
    """run() on 64-pixel tiles (the default) and on 128-pixel tiles; returns (narrow results, kernel name), after checking
    that every result is bit-identical between the two and both launches ran the same kernel variant."""
    got = {}
    try:
        for narrow in (0, 1):
            _lib.set_tuning("conv_narrow", narrow)
            res = run()
            torch.cuda.synchronize()
            got[narrow] = ([r.cpu().numpy() for r in res], _lib.last_kernel())
    finally:
        _lib.set_tuning("conv_narrow", 1)
    (wide, k0), (narrow, k1) = got[0], got[1]
    assert k0 == k1, (k0, k1)
    for a, b in zip(narrow, wide):
        assert np.array_equal(a, b, equal_nan=True), (k1, float(np.nanmax(np.abs(a - b))))
    return narrow, k1


def close(got, ref, tol=1e-4):
    err = float(np.abs(got - ref).max())
    assert err <= tol * max(1.0, float(np.abs(ref).max())), err


# ------------------------------------------------------------------------------------------------------------------
# CPU: the split-K plans do not depend on the tile width
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("W", WIDTHS + [65])
def test_plans_count_one_tile_column_of_two_rows(W):
    """An output at most 64 pixels wide is one tile column in either geometry, so plan_split (host arithmetic) sees the
    same N * ceil(OH / 2) tiles and returns the same workspace with 64- or 128-pixel tile rows."""
    wb = _lib.lib().mfn_conv3x3_workspace_bytes
    shapes = [(1, 451, 28, W, 96, 1, 1), (8, 675, 14, W, 64, 1, 1), (8, 529, 7, W, 64, 1, 1), (2, 100, 9, W, 48, 1, 1),
              (16, 128, 28, 2 * W, 196, 2, 1), (1, 96, 16, W, 64, 1, 16)]
    try:
        for s in shapes:
            _lib.set_tuning("conv_narrow", 1)
            a = wb(*s)
            _lib.set_tuning("conv_narrow", 0)
            assert wb(*s) == a, s
            N, Cin, H, Wi, Cout, stride, _ = s
            OH, OW = (H - 1) // stride + 1, (Wi - 1) // stride + 1
            tiles = N * -(-OW // 128) * -(-OH // 2)
            ns = 2 if Cout > 128 else 1
            chunks = (Cin + 15) // 16
            if 2 * tiles * ns <= 132:      # every tile split: min(132 // (tiles ns), chunks // 3, 8) parts
                k = min(132 // (tiles * ns), chunks // 3, 8)
                assert a == (4 * k * N * Cout * OH * OW if k >= 2 else 0), s
    finally:
        _lib.set_tuning("conv_narrow", 1)


# ------------------------------------------------------------------------------------------------------------------
# GPU: fp32 NCHW input (the producer warps convert it)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("W", WIDTHS)
@pytest.mark.parametrize("case", ["plain", "dil2_prefix", "d2s", "stride2", "splitk", "grid_cap"])
def test_fp32_input(W, case):
    rng = np.random.default_rng(1000 + W + 17 * len(case))
    N, Cin, H, Cout, dil, stride, d2s, lin = 2, 40, 9, 35, 1, 1, False, 0
    if case == "dil2_prefix":
        dil, lin, Cout = 2, 3, 72
    elif case == "d2s":
        d2s, Cout = True, 48
    elif case == "stride2":
        stride, Cout = 2, 64
    elif case == "splitk":
        Cin, Cout, H = 100, 96, 7
    elif case == "grid_cap":
        Cout, H = 128, 13
    Wi = 2 * W - (W % 2) if stride == 2 else W
    x = feat(rng, (N, Cin, H, Wi))
    w, b = weights(rng, Cout, Cin, Cout // 4 if d2s else None)
    if case == "splitk":
        assert _lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, Wi, Cout, 1, 1) > 0
    OH, OW = (H - 1) // stride + 1, (Wi - 1) // stride + 1
    F = Cout // 4 if d2s else Cout
    s = 2 if d2s else 1
    xg, pk, bg = cu(x), ops.conv3x3_pack(cu(w)), cu(b)

    def run():
        out = torch.full((N, F + 3, s * OH, s * OW), float("nan"), device=DEV)
        ops.conv3x3_slices(xg, 0, Cin, pk, bg, out, 2, Cout, 0.1, dilation=dil, stride=stride, depth_to_space=d2s,
                           linear_prefix=lin)
        return [out]

    if case == "grid_cap":
        _lib.set_tuning("conv_grid_cap", 3)
    try:
        (out,), kern = both(run)
    finally:
        _lib.set_tuning("conv_grid_cap", 0)
    want = "conv3x3_wgmma_reduce_kernel" if case == "splitk" else f"conv3x3_wgmma_kernel<CoutP={(Cout + 15) // 16 * 16}"
    assert kern.startswith(want), kern
    assert np.isnan(out[:, :2]).all() and np.isnan(out[:, 2 + F:]).all(), kern
    close(out[:, 2:2 + F], reference(x, w, b, dil, stride, d2s, lin))


# ------------------------------------------------------------------------------------------------------------------
# GPU: split input (tensor copies), split output, linear-prefix heads, depth-to-space, bf16
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("W", WIDTHS)
@pytest.mark.parametrize("case", ["dil1", "dil2_split_out", "dil4_split_out", "heads", "d2s", "splitk_split_out",
                                  "bf16_split_out", "bf16_heads"])
def test_split_input(W, case):
    rng = np.random.default_rng(2000 + W + 31 * len(case))
    N, H, Cin, Cout, dil, lin, d2s = 2, 9, 70, 32, 1, 0, False
    bf16 = case.startswith("bf16")
    split_out = "split_out" in case
    if case.startswith("dil2"):
        dil = 2
    elif case.startswith("dil4"):
        dil = 4
    elif case.endswith("heads"):
        lin, Cout = 4, 36          # 3 linear heads (+ one zero pad channel) in front of 32 activated channels
        split_out = True
    elif case == "d2s":
        d2s, Cout = True, 64
    elif case.startswith("splitk"):
        Cin, H = 100, 7
    elif case == "dil1":
        Cout = 48
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin, Cout // 4 if d2s else None)
    if lin:
        w[lin - 1] = 0.0
        b[:lin] = 0.0
    c_in0 = 16                      # the input slice starts one 16-channel group into the buffer
    act = ops.SplitAct(N, c_in0 + Cin, H, W, DEV, bf16=bf16)
    act.pack(cu(x), c_in0)
    pk, bg = ops.conv3x3_pack(cu(w)), cu(b)
    Fo = Cout - lin

    def run():
        res = []
        if split_out:
            dst = ops.SplitAct(N, 16 + Fo + 16, H, W, DEV, bf16=bf16)
            dst.buf.fill_(0x7F)     # pattern: channels outside the written slice must keep it
            pre = torch.full((N, lin, H, W), float("nan"), device=DEV) if lin else None
            ops.conv3x3_split(act, c_in0, Cin, pk, bg, Cout, 0.1, dil, out=pre, out_split=dst, out_c0=16,
                              linear_prefix=lin, bf16=bf16)
            res.append(dst.buf)
            if lin:
                res.append(pre)
        else:
            s = 2 if d2s else 1
            out = torch.full((N, Cout // 4 if d2s else Cout, s * H, s * W), float("nan"), device=DEV)
            ops.conv3x3_split(act, c_in0, Cin, pk, bg, Cout, 0.1, dil, out=out, depth_to_space=d2s, bf16=bf16)
            res.append(out)
        return res

    res, kern = both(run)
    if case.startswith("splitk"):      # the last launch is the split-K reduction
        assert kern == "conv3x3_wgmma_reduce_kernel", kern
    else:
        assert kern.startswith(f"conv3x3_wgmma_kernel<CoutP={(Cout + 15) // 16 * 16}"), kern
        assert kern.endswith(",bf16>") == bf16, kern
    ref = reference(x, w, b, dil, 1, d2s, lin)
    tol = 2e-2 if bf16 else 1e-4
    if split_out:
        buf = res[0]
        dst = ops.SplitAct(N, 16 + Fo + 16, H, W, DEV, bf16=bf16)
        dst.buf.copy_(torch.from_numpy(buf))
        hi, lo = dst.hi_lo()
        got = (hi.double() + lo.double()).cpu().numpy()
        close(got[:, 16:16 + Fo], ref[:, lin:], tol)
        pattern = np.full(16, 0x7F, np.uint8)
        groups = buf.reshape(N, buf.shape[1], -1, H * W, 16)
        assert (groups[:, :, :2] == pattern).all() and (groups[:, :, 2 + Fo // 8:] == pattern).all(), kern
        if lin:
            close(res[1], ref[:, :lin], tol)
    else:
        close(res[0], ref, tol)
