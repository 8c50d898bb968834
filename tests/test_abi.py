"""The C-ABI library loads and exports every symbol include/maskflow_b200.h declares; argument validation works without a
GPU (no compute is launched here)."""
import ctypes
import os
import re

import pytest

from maskflownet_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "maskflow_b200.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"MFN_API\s+([\w\s\*]+?)\s*\b(mfn_\w+)\s*\(([^;]*?)\)\s*;", src, flags=re.S):
        args = [a.strip() for a in m.group(3).replace("\n", " ").split(",")]
        out[m.group(2)] = [a for a in args if a and a != "void"]
    return out


TUNING_KEYS = {"corr_grid_cap", "corr_tma", "corr_rb", "warp_lin", "conv_wgmma", "conv_grid_cap", "conv_splitk",
               "conv_narrow", "conv_tma_in", "conv_dbg"}
RETIRED_TUNING_KEYS = ("corr_ts_lo", "corr_ts_hi", "corr_disable_ring", "corr_ring_th", "corr_dbg", "corr_rb_twb",
                       "corr_rb_rows", "warp_lin_fch", "conv_as", "conv_wgmma_min_w")


def documented_tuning_keys():
    """{key: default} from the list in the comment above mfn_set_tuning."""
    src = open(HEADER).read()
    block = re.search(r"/\*((?:(?!/\*).)*?)\*/\s*MFN_API int mfn_set_tuning", src, flags=re.S).group(1)
    return {k: int(v) for k, v in re.findall(r'^\s*\*\s+"(\w+)"\s+default (-?\d+):', block, flags=re.M)}


def struct_tuning_defaults():
    """{field: default} of mfn::Tuning (csrc/common.cuh)."""
    src = open(os.path.join(ROOT, "maskflownet_b200", "csrc", "common.cuh")).read()
    body = re.search(r"struct Tuning \{(.*?)\};", src, flags=re.S).group(1)
    return {k: int(v) for k, v in re.findall(r"int (\w+) = (-?\d+);", body)}


def test_every_declared_symbol_is_exported():
    decl = declared_functions()
    assert len(decl) >= 16
    L = _lib.lib()
    for name in decl:
        assert hasattr(L, name), f"{name} declared in the header but not exported by {_lib.SO_PATH}"
    assert L.mfn_version() == 100


def test_ctypes_table_matches_header():
    decl = declared_functions()
    for name, argtypes in _lib.SIGNATURES.items():
        assert name in decl, name
        assert len(argtypes) == len(decl[name]), (name, len(argtypes), decl[name])
        for a, ct in zip(decl[name], argtypes):
            if "*" in a and "char" not in a:
                assert ct is ctypes.c_void_p, (name, a)
            elif a.startswith("long long"):
                assert ct is ctypes.c_longlong, (name, a)
            elif a.startswith("float"):
                assert ct is ctypes.c_float, (name, a)
            elif a.startswith("int"):
                assert ct is ctypes.c_int, (name, a)
    ops_in_header = {n for n in decl if n not in ("mfn_version", "mfn_last_error", "mfn_last_kernel", "mfn_launch_count",
                                               "mfn_conv3x3_packed_bytes", "mfn_warp_resample_workspace_bytes",
                                               "mfn_conv3x3_workspace_bytes", "mfn_color_augment_workspace_bytes",
                                               "mfn_multiscale_epe_workspace_bytes")}
    assert ops_in_header == set(_lib.SIGNATURES), ops_in_header ^ set(_lib.SIGNATURES)


def test_argument_errors_need_no_gpu():
    L = _lib.lib()
    rc = L.mfn_correlation_forward(None, None, None, 1, 1, 1, 1, 4, 1, 4, 1, 1, 1, 0, 1.0, 0, None)
    assert rc == -1 and b"null pointer" in L.mfn_last_error()
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    rc = L.mfn_correlation_forward(p, p, p, 1, 1, 2, 2, 4, 2, 4, 1, 1, 1, 0, 1.0, 0, None)   # even kernel_size
    assert rc == -1 and b"odd" in L.mfn_last_error()
    rc = L.mfn_correlation_forward(p, p, p, 1, 1, 2, 2, 4, 1, 4, 2, 1, 1, 0, 1.0, 3, None)   # MMA kernel, stride1=2
    assert rc == -2
    rc = L.mfn_deformable_conv_forward(p, p, p, None, p, 1, 1, 2, 2, 1, 5, 5, 1, 1, 1, 1, 2, 2, 1, 1, 0, None)
    assert rc == -2 and b"3x3" in L.mfn_last_error()
    rc = L.mfn_warp_mask_forward(p, p, None, p, None, None, p, None, None, None, 1, 1, 3, 3, 1, 2, 20.0, 4.0, 0.1, 0, None)
    assert rc == -1 and b"multiples" in L.mfn_last_error()
    with pytest.raises(_lib.MaskflowError):
        _lib.set_tuning("no_such_key", 1)
    # the header's list of tuning keys is the set the library accepts, with the defaults the library starts from
    documented = documented_tuning_keys()
    assert set(documented) == TUNING_KEYS, set(documented) ^ TUNING_KEYS
    assert documented == struct_tuning_defaults()
    for key, default in documented.items():
        _lib.set_tuning(key, default)
    for key in RETIRED_TUNING_KEYS:
        with pytest.raises(_lib.MaskflowError, match="unknown key"):
            _lib.set_tuning(key, 0)
    assert _lib.launch_count() == 0 or _lib.launch_count() >= 0


def test_conv_split_plan_is_host_arithmetic():
    """mfn_conv3x3_workspace_bytes is pure host arithmetic (no GPU): the split-K plan of the wgmma convolution for the
    shapes of BASELINE configs[1] (csrc/conv3x3_wgmma.cu: plan_split)."""
    L = _lib.lib()
    wb = L.mfn_conv3x3_workspace_bytes
    # level 6 (7x16, N=8: 32 tiles): every tile split into min(132 // 32, 34 // 3, 8) = 4 parts over the whole tensor
    assert wb(8, 529, 7, 16, 64, 1, 1) == 4 * 8 * 64 * 7 * 16 * 4
    # level 5 (14x32, N=8: 56 tiles): 2 parts
    assert wb(8, 675, 14, 32, 64, 1, 1) == 2 * 8 * 64 * 14 * 32 * 4
    # level 2, long tensor-bound layer at batch 6: 672 tiles = 5 x 132 + 12 -> the last 12 tiles (12 rows of the last
    # sample) in min(132 // 12, 37 // 2) = 11 parts; at batch 8 (896 = 6 x 132 + 104) the last round is nearly full: no split
    assert wb(6, 579, 112, 256, 128, 1, 1) == 11 * 1 * 128 * 12 * 256 * 4
    assert wb(8, 579, 112, 256, 128, 1, 1) == 0
    # same geometry but few chunks / narrow output: not worth a second launch
    assert wb(6, 128, 112, 256, 128, 1, 1) == 0
    assert wb(6, 547, 112, 256, 34, 1, 1) == 0
    # levels 3 and 4 (224 / 112 tiles), the pyramid (thousands of tiles) and nonsense arguments: never split
    assert wb(8, 419, 56, 128, 96, 1, 1) == 0 and wb(8, 451, 28, 64, 96, 1, 1) == 0
    assert wb(16, 16, 224, 512, 16, 1, 1) == 0 and wb(16, 3, 448, 1024, 16, 2, 1) == 0
    assert wb(0, 16, 8, 8, 16, 1, 1) == 0 and wb(8, 16, 8, 8, 300, 1, 1) == 0
