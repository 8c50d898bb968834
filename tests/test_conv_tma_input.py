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

from launchcheck.conv_tma import check, feat, run_both, weights


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
