"""The wgmma convolution's TMA-staged fp32 input at stride 2 (csrc/conv3x3_wgmma.cu, SplitDev::in == 2): one thread copies
each 8-channel plane of a chunk's raw input rows into shared memory with a tensor copy, and the producer warps
de-interleave it from there into the even / odd entries they used to load pixel by pixel.  Stride 2 then runs 64-pixel
tile rows.  The MMAs see the same entries in the same order, so every launch is compared bit for bit with the per-thread
loads on 128-pixel tiles (tuning knob conv_tma_in = 0) and against a float64 convolution.  Covered: the pyramid's
stride-2 layers at the benchmark's shapes and the cascade's 4-channel input, odd and even image sizes with the box
meeting the right edge at every position, Cin 3 to 40, a channel slice of a wider buffer, capped grids, both product
modes, and the shapes the host keeps on the per-thread loads (widths not a multiple of 4, an unaligned input, outputs at
most 64 wide).  Also: the pyramid reads ops.preprocess's two images as one batch without a copy, with the same flow."""
import numpy as np
import pytest
import torch

from maskflownet_b200 import _lib, network, ops

from launchcheck.conv_tma import check, feat, run_both, weights
from launchcheck.inputs import _deterministic, _same

# (N, Cin, Cout, H, W): conv1a / conv2a / conv3a at the benchmark's size (both images, batch 8), and the cascade's conv1x
# (its 4-channel input, batch 4, one image per pyramid pass)
BENCH = {"conv1a": (16, 3, 16, 448, 1024), "conv2a": (16, 16, 32, 224, 512), "conv3a": (16, 32, 64, 112, 256),
         "conv1x": (4, 4, 16, 448, 1024)}


def test_stride2_layers_are_not_split():
    """The stride-2 layers of the benchmark run without split-K on their 64-pixel tiles (host arithmetic, no GPU)."""
    wb = _lib.lib().mfn_conv3x3_workspace_bytes
    for N, Cin, Cout, H, W in BENCH.values():
        assert wb(N, Cin, H, W, Cout, 2, 1) == 0, (N, Cin, Cout, H, W)


@pytest.mark.gpu
@pytest.mark.parametrize("layer", sorted(BENCH))
def test_bench_stride2_layers(layer):
    N, Cin, Cout, H, W = BENCH[layer]
    rng = np.random.default_rng(sum(map(ord, layer)))
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, 0, Cin, w, b, stride=2)
    n = 2   # float64 on two samples keeps the CPU reference short; the bitwise comparison covered all of them
    check(got[:n], x[:n], w, b, stride=2)


@pytest.mark.gpu
@pytest.mark.parametrize("H", [5, 8])
@pytest.mark.parametrize("Cin", [3, 4, 16, 19, 32, 40])
@pytest.mark.parametrize("W", [64, 130, 131, 132, 136, 200, 256, 260, 300])
def test_borders_and_partial_chunks(W, Cin, H):
    """Padding on all four sides, odd and even sizes: a tile's box spans input pixels 2 x0 - 4 .. 2 x0 + 127, and these
    widths put the image's right edge 4 to 128 pixels into the last one.  Cin <= 8 loads one plane per chunk, the others
    two (the channels past Cin read zero).  W = 130, 131 (not multiples of 4) and W = 64 (a 32-pixel output) keep the
    per-thread loads."""
    rng = np.random.default_rng(1000 * H + 10 * Cin + W)
    N, Cout = 2, 48
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, 0, Cin, w, b, stride=2)
    check(got, x, w, b, stride=2)


@pytest.mark.gpu
@pytest.mark.parametrize("c0", [4, 20])
def test_channel_slice_of_a_wider_buffer(c0):
    """Channels [c0, c0 + Cin) of a buffer with more channels on both sides: nothing outside the slice enters the sums."""
    rng = np.random.default_rng(c0)
    N, C, Cin, H, W, Cout = 3, 70, 19, 7, 264, 32
    x = feat(rng, (N, C, H, W))
    x[:, :c0] = 1e6
    x[:, c0 + Cin:] = -1e6
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, c0, Cin, w, b, stride=2)
    check(got, x[:, c0:c0 + Cin], w, b, stride=2)


@pytest.mark.gpu
def test_unaligned_input_keeps_the_per_thread_loads():
    """An input 4 bytes into its allocation has no tensor map: the launch must take the per-thread loads, correctly."""
    rng = np.random.default_rng(5)
    N, Cin, H, W, Cout = 2, 16, 9, 260, 32
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin)
    got, _, _ = run_both(x, 0, Cin, w, b, stride=2, shift=1)
    check(got, x, w, b, stride=2)


@pytest.mark.gpu
@pytest.mark.parametrize("cap", [1, 3])
@pytest.mark.parametrize("bf16", [False, True])
@pytest.mark.parametrize("Cin", [3, 40])
def test_capped_grids_and_bf16(Cin, cap, bf16):
    """Long per-CTA runs of tiles (the raw ring refills across chunk and tile boundaries, one or two stages per chunk) in
    both product modes."""
    rng = np.random.default_rng(Cin + cap + 10 * bf16)
    N, H, W, Cout = 2, 11, 400, 64
    x = feat(rng, (N, Cin, H, W))
    w, b = weights(rng, Cout, Cin)
    got, k1, _ = run_both(x, 0, Cin, w, b, stride=2, bf16=bf16, grid_cap=cap)
    assert k1.endswith(",bf16>") == bf16, k1
    check(got, x, w, b, stride=2, bf16=bf16)


@pytest.mark.gpu
def test_pyramid_reads_the_preprocessed_pair_without_a_copy():
    """ops.preprocess returns its two images as adjacent halves of one buffer, and the forward on them (the pyramid reads
    the buffer as one batch) equals, bit for bit, the forward on two separate tensors (the pyramid concatenates them)."""
    g = torch.Generator().manual_seed(3)
    u1 = torch.randint(0, 256, (2, 3, 128, 256), dtype=torch.uint8, generator=g).cuda()
    u2 = torch.randint(0, 256, (2, 3, 128, 256), dtype=torch.uint8, generator=g).cuda()
    torch.manual_seed(0)
    model = network.MaskFlownetS().cuda().eval()
    with _deterministic(), torch.no_grad():
        a, b, _ = ops.preprocess(u1, u2)
        assert a.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()
        assert b.storage_offset() == a.storage_offset() + a.numel()
        got = model(a, b)[0][-1].clone()
        ref = model(a.clone(), b.clone())[0][-1]
    _same(got, ref, "preprocessed pair")
