"""ctypes binding of libmaskflow_b200.so (C ABI declared in include/maskflow_b200.h).

The library is the product: there is NO CPU or PyTorch fallback.  If the shared object is missing, or a call is made
without CUDA tensors, this module raises -- loudly -- instead of computing something else.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("MFN_LIB_PATH") or os.path.join(_HERE, "libmaskflow_b200.so")   # MFN_LIB_PATH: A/B experiments
_lib = None

_f = ctypes.c_void_p  # device pointers travel as integers
_i = ctypes.c_int
_ll = ctypes.c_longlong
_fl = ctypes.c_float

# name -> argtypes; mirrors include/maskflow_b200.h one to one (tests/test_abi.py checks header <-> table <-> .so)
SIGNATURES = {
    "mfn_correlation_forward": [_f, _f, _f, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _ll, _fl, _i, _f],
    "mfn_correlation_backward": [_f, _f, _f, _f, _f, _f, _i, _i, _i, _i, _i, _ll, _fl, _f],
    "mfn_deformable_conv_forward": [_f, _f, _f, _f, _f] + [_i] * 16 + [_f],
    "mfn_deformable_conv_backward": [_f] * 8 + [_i] * 6 + [_f],
    "mfn_warp_mask_forward": [_f] * 10 + [_i] * 6 + [_fl, _fl, _fl, _i, _f],
    "mfn_warp_mask_forward_tc": [_f] * 10 + [_i] * 6 + [_fl, _fl, _fl, _i, _f],
    "mfn_warp_mask_forward_resample": [_f] * 11 + [_i] * 6 + [_fl, _fl, _fl, _i, _f],
    "mfn_warp_mask_backward": [_f] * 14 + [_i] * 5 + [_fl, _fl, _fl, _i, _f],
    "mfn_upsample_forward": [_f, _f, _i, _i, _i, _i, _fl, _f],
    "mfn_upsample_backward": [_f, _f, _i, _i, _i, _i, _fl, _f],
    "mfn_grid_generator_warp_forward": [_f, _f, _i, _i, _i, _f],
    "mfn_bilinear_sampler_forward": [_f, _f, _f, _i, _i, _i, _i, _i, _i, _f],
    "mfn_image_warp_concat_forward": [_f] * 6 + [_i] * 4 + [_fl, _f],
    "mfn_grid_generator_warp_backward": [_f, _f, _i, _i, _i, _f],
    "mfn_bilinear_sampler_backward": [_f] * 5 + [_i] * 6 + [_f],
    "mfn_image_warp_concat_backward": [_f] * 7 + [_i] * 4 + [_fl, _f],
    "mfn_preprocess_forward": [_f, _f, _i, _f, _f, _f, _i, _i, _i, _i, _i, _i, _f],
    "mfn_postprocess_forward": [_f, _f, _i, _i, _i, _i, _i, _i, _i, _i, _f],
    "mfn_flow_to_color": [_f, _f, _f, _i, _i, _i, _fl, _i, _f],
    "mfn_warp_mask_backward_det": [_f] * 14 + [_i] * 5 + [_fl, _fl, _fl, _i, _f, _ll, _f],
    "mfn_deformable_conv_backward_det": [_f] * 8 + [_i] * 6 + [_f, _ll, _f],
    "mfn_bilinear_sampler_backward_det": [_f] * 5 + [_i] * 6 + [_f, _ll, _f],
    "mfn_image_warp_concat_backward_det": [_f] * 7 + [_i] * 4 + [_fl, _f, _ll, _f],
    "mfn_preprocess_forward_det": [_f, _f, _i, _f, _f, _f, _i, _i, _i, _i, _i, _i, _f, _ll, _f],
    "mfn_geometry_augment_forward": [_f, _f, _i, _f, _f, _i, _f, _f, _f, _f, _f, _i, _i, _i, _i, _i, _f],
    "mfn_color_augment_forward": [_f, _f, _f, _f, _f, _fl, _ll, _f, _f, _f, _ll, _i, _i, _i, _i, _f],
    "mfn_multiscale_epe_forward": [_f, _f, _f, _f, _f, _i, _fl, _fl, _f, _f, _f, _ll, _i, _i, _i, _f],
    "mfn_multiscale_epe_backward": [_f, _f, _f, _f, _f, _i, _fl, _fl, _f, _f, _f, _i, _i, _i, _f],
    "mfn_set_tuning": [ctypes.c_char_p, _i],
    "mfn_conv3x3_pack_weights": [_f, _f, _i, _i, _f],
    "mfn_conv3x3_forward": [_f, _ll, _f, _f, _f, _ll, _i, _i, _i, _i, _i, _i, _fl, _f],
    "mfn_conv3x3_forward_ex": [_f, _ll, _f, _f, _f, _ll, _i, _i, _i, _i, _i, _i, _i, _i, _fl, _f],
    "mfn_conv3x3_forward_ws": [_f, _ll, _f, _f, _f, _ll, _i, _i, _i, _i, _i, _i, _i, _i, _fl, _f, _ll, _f],
}


class MaskflowError(RuntimeError):
    pass


def build(verbose: bool = False) -> str:
    """Compile the CUDA sources in-tree with nvcc for sm_90a (no GPU needed).  Returns the .so path."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    res = subprocess.run(cmd, capture_output=not verbose, text=True)
    if res.returncode != 0:
        raise MaskflowError("building libmaskflow_b200.so failed:\n" + (res.stdout or "") + (res.stderr or ""))
    return SO_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise MaskflowError(
                f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C maskflownet_b200/csrc`).  There is no CPU / PyTorch fallback for the hot path.")
        L = ctypes.CDLL(SO_PATH)
        L.mfn_version.restype = ctypes.c_int
        L.mfn_last_error.restype = ctypes.c_char_p
        L.mfn_last_kernel.restype = ctypes.c_char_p
        L.mfn_launch_count.restype = ctypes.c_ulonglong
        L.mfn_conv3x3_packed_bytes.restype = ctypes.c_longlong
        L.mfn_conv3x3_packed_bytes.argtypes = [ctypes.c_int, ctypes.c_int]
        L.mfn_conv3x3_workspace_bytes.restype = ctypes.c_longlong
        L.mfn_conv3x3_workspace_bytes.argtypes = [ctypes.c_int] * 7
        L.mfn_color_augment_workspace_bytes.restype = ctypes.c_longlong
        L.mfn_color_augment_workspace_bytes.argtypes = [ctypes.c_int]
        L.mfn_multiscale_epe_workspace_bytes.restype = ctypes.c_longlong
        L.mfn_multiscale_epe_workspace_bytes.argtypes = [ctypes.c_int]
        L.mfn_warp_resample_workspace_bytes.restype = ctypes.c_longlong
        L.mfn_warp_resample_workspace_bytes.argtypes = [ctypes.c_int] * 4
        for name, argtypes in SIGNATURES.items():
            fn = getattr(L, name)
            fn.argtypes = argtypes
            fn.restype = ctypes.c_int
        _lib = L
        # experiment hook: MFN_TUNING="key=value,key=value" applies mfn_set_tuning at load time
        for item in filter(None, os.environ.get("MFN_TUNING", "").split(",")):
            key, _, val = item.partition("=")
            if key.strip() == "corr_dbg":
                # the phase-ablation switches produce INVALID results: tools set them through set_tuning(), never the environment
                raise MaskflowError("MFN_TUNING: corr_dbg is a profiling switch (results invalid); set it from a tool, not the environment")
            if L.mfn_set_tuning(key.strip().encode(), int(val)):
                raise MaskflowError(f"MFN_TUNING: {L.mfn_last_error().decode()}")
    return _lib


def last_error() -> str:
    return lib().mfn_last_error().decode()


def last_kernel() -> str:
    return lib().mfn_last_kernel().decode()


def launch_count() -> int:
    return int(lib().mfn_launch_count())


def call(name: str, *args) -> None:
    rc = getattr(lib(), name)(*args)
    if rc != 0:
        kind = "argument/support error" if rc < 0 else "CUDA error"
        raise MaskflowError(f"{name} failed ({kind} {rc}): {last_error()}")


def set_tuning(key: str, value: int) -> None:
    call("mfn_set_tuning", key.encode(), int(value))
