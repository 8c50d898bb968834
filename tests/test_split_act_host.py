"""The split-activation pack kernel (csrc/split_act.cu) compiled for the host (tests/host_emu/split_act_emu.cpp) against a
numpy restatement of the format: for every fp32 value v, hi = bf16 round-to-nearest-even of v and lo = that of v - hi, in
(N, 2, Cg, H, W, 8) bf16 with zero pad channels; partial 8- and 16-channel groups, NaN / inf / overflow, a slice that
starts inside a larger buffer and a batch stride wider than the tensor.  No GPU."""
import ctypes

import numpy as np
import pytest

from launchcheck.emu import build


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "split_act_emu")
    L.emu_split_pack.argtypes = [ctypes.c_void_p, ctypes.c_longlong] + [ctypes.c_int] * 4 + [ctypes.c_void_p] + \
        [ctypes.c_int] * 2
    L.emu_split_pack.restype = None
    return L


def bf16_rn(x):
    """fp32 -> bf16 bits, round to nearest even (NaN handled by the caller)."""
    u = x.astype(np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_value(h):
    return (h.astype(np.uint32) << 16).view(np.float32)


def expected(src, dst_channels, dst_c0):
    """The whole split buffer (uint16, (N, 2, Cg, H, W, 8)) after packing src at dst_c0 into a zeroed buffer."""
    N, C, H, W = src.shape
    Cg = (dst_channels + 15) // 16 * 2
    with np.errstate(invalid="ignore", over="ignore"):
        hi = bf16_rn(src)
        lo = bf16_rn(src - bf16_value(hi))
    out = np.zeros((N, 2, Cg * 8, H, W), np.uint16)
    out[:, 0, dst_c0:dst_c0 + C], out[:, 1, dst_c0:dst_c0 + C] = hi, lo
    return out.reshape(N, 2, Cg, 8, H, W).transpose(0, 1, 2, 4, 5, 3)


def pack(emu, x, dst_channels, dst_c0, C=None):
    """Channels [0, C) of x (default: all) into a zeroed buffer of dst_channels channels at dst_c0."""
    N, Cx, H, W = x.shape
    C = C or Cx
    Cg = (dst_channels + 15) // 16 * 2
    buf = np.zeros((N, 2, Cg, H, W, 8), np.uint16)
    emu.emu_split_pack(x.ctypes.data_as(ctypes.c_void_p), Cx * H * W, N, C, H, W,
                       buf.ctypes.data_as(ctypes.c_void_p), dst_channels, dst_c0)
    return buf


def check(got, want):
    """Bit-equal, except that a NaN only has to be a NaN (numpy keeps payloads, the instruction writes the canonical NaN)."""
    gn, wn = np.isnan(bf16_value(got)), np.isnan(bf16_value(want))
    assert np.array_equal(gn, wn)
    assert np.array_equal(np.where(gn, 0, got), np.where(wn, 0, want))


@pytest.mark.parametrize("C,dst_channels,dst_c0", [(35, 35, 0), (35, 51, 16), (5, 21, 16), (32, 80, 32), (131, 579, 448)])
def test_pack_matches_numpy(emu, C, dst_channels, dst_c0):
    rng = np.random.default_rng(C)
    x = (rng.standard_normal((2, C, 3, 7)) * np.exp2(rng.integers(-30, 30, (2, C, 3, 7)))).astype(np.float32)
    check(pack(emu, x, dst_channels, dst_c0), expected(x, dst_channels, dst_c0))


def test_pack_special_values(emu):
    x = np.array([np.nan, np.inf, -np.inf, 3.4e38, -3.4e38, 0.0, -0.0, 1e-40, -1e-45, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8,
                  65504.0, 1.00390625, np.float32(np.pi)], np.float32)
    x = np.tile(x, 3)[:37].reshape(1, 37, 1, 1)
    got = pack(emu, x, 37, 0)
    check(got, expected(x, 37, 0))
    v = bf16_value(got).transpose(0, 1, 2, 5, 3, 4).reshape(2, -1)
    assert v[0, 1] == np.inf and np.isnan(v[1, 1])            # inf: hi inf, lo inf - inf
    assert v[0, 3] == np.inf and v[1, 3] == -np.inf           # 3.4e38 rounds past the largest bf16
    assert v[0, 9] == 1.0 and v[0, 10] == 1.0 + 4 * 2.0 ** -8  # ties to even


def test_pack_honours_batch_stride(emu):
    rng = np.random.default_rng(3)
    full = rng.standard_normal((2, 20, 4, 5)).astype(np.float32)
    got = pack(emu, full, 16, 0, C=16)   # channels 0..15 of each 20-channel sample
    check(got, expected(np.ascontiguousarray(full[:, :16]), 16, 0))
