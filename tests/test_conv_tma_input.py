"""The wgmma convolution's TMA-staged fp32 input (csrc/conv3x3_wgmma.cu, SplitDev::in == 2): at stride 1 and dilation 1
one thread copies each chunk's raw fp32 tile into shared memory with a tensor copy, and the producer warps convert it from
there instead of loading it pixel by pixel.  The converted stage holds the same entries in the same layout and the MMAs
run in the same order, so every launch is compared bit for bit with the per-thread loads (tuning knob conv_tma_in = 0)
and against a float64 convolution.  Covered: the pyramid shapes of the benchmark, image borders, channel slices of a
wider buffer, Cin not a multiple of 16, split-K, capped grids, the bf16 mode, and the shapes the host keeps on the
per-thread loads (widths not a multiple of 4, an unaligned input, stride 2, dilation 2, outputs at most 64 wide).  Both input paths share the
kernel's variant name (they compute the same sums in the same order), so these tests pin the results, not the choice."""
import numpy as np
import pytest
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


# (N, Cin, Cout, H, W): conv1b / conv2b / conv3b at the benchmark's size (both images, batch 8), and the level 4-6 layers,
# whose 64-pixel tiles keep the per-thread loads
BENCH = {"conv1b": (16, 16, 16, 224, 512), "conv2b": (16, 32, 32, 112, 256), "conv3b": (16, 64, 64, 56, 128),
         "conv4b": (16, 96, 96, 28, 64), "conv5b": (16, 128, 128, 14, 32), "conv6b": (16, 196, 196, 7, 16)}


@pytest.mark.gpu
@pytest.mark.parametrize("layer", sorted(BENCH))
def test_bench_pyramid_layers(layer):
    N, Cin, Cout, H, W = BENCH[layer]
    rng = np.random.default_rng(sum(map(ord, layer)))
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, 0, Cin, w, b)
    n = 2   # float64 on two samples keeps the CPU reference short; the bitwise comparison covered all of them
    check(got[:n], x[:n], w, b)


@pytest.mark.gpu
@pytest.mark.parametrize("Cin", [3, 4, 16, 40, 131])
@pytest.mark.parametrize("W", [4, 60, 64, 128, 132, 260])
def test_borders_and_partial_chunks(Cin, W):
    """Padding on all four sides (the image is a few tiles, its edges at every position of a box), Cin not a multiple of
    16 (the channels past Cin read zero from the tensor map), one and several tile columns."""
    rng = np.random.default_rng(7 * Cin + W)
    N, H, Cout = 2, 5, 48
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, 0, Cin, w, b)
    check(got, x, w, b)


@pytest.mark.gpu
@pytest.mark.parametrize("c0", [4, 20])
def test_channel_slice_of_a_wider_buffer(c0):
    """Channels [c0, c0 + Cin) of a buffer with more channels on both sides: nothing outside the slice enters the sums."""
    rng = np.random.default_rng(c0)
    N, C, Cin, H, W, Cout = 3, 70, 19, 6, 136, 32
    x = feat(rng, (N, C, H, W))
    x[:, :c0] = 1e6
    x[:, c0 + Cin:] = -1e6
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, c0, Cin, w, b)
    check(got, x[:, c0:c0 + Cin], w, b)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [1, 3])
@pytest.mark.parametrize("bf16", [False, True])
def test_capped_grids_and_bf16(cap, bf16):
    """Long per-CTA runs of tiles (the raw ring refills across tile boundaries) in both product modes."""
    rng = np.random.default_rng(cap + 10 * bf16)
    N, Cin, H, W, Cout = 2, 40, 9, 200, 64
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin)
    got, k1, _ = run_both(x, 0, Cin, w, b, bf16=bf16, grid_cap=cap)
    assert k1.endswith(",bf16>") == bf16, k1
    check(got, x, w, b, bf16=bf16)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["odd_width", "width_mod4_2", "unaligned_slice", "stride2", "dil2"])
def test_shapes_that_keep_the_per_thread_loads(case):
    """The host takes the tensor map only where it is valid: row and sample strides that are 16-byte multiples (W % 4 == 0),
    a 16-byte aligned slice start, stride 1 and dilation 1.  Elsewhere the launch must run the per-thread loads, and
    correctly: a tensor map over such an input would fail to encode or read the wrong pixels."""
    rng = np.random.default_rng(len(case))
    N, C, c0, Cin, H, W, Cout, stride, dil, shift = 2, 24, 0, 24, 7, 132, 32, 1, 1, 0
    if case == "odd_width":
        W = 131
    elif case == "width_mod4_2":
        W = 130
    elif case == "unaligned_slice":
        shift = 1   # the buffer starts 4 bytes into its allocation: no channel slice of it is 16-byte aligned
    elif case == "stride2":
        stride = 2
    else:
        dil = 2
    x = feat(rng, (N, C, H, W))
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, c0, Cin, w, b, stride=stride, dil=dil, shift=shift)
    check(got, x[:, c0:c0 + Cin], w, b, stride=stride, dil=dil)
