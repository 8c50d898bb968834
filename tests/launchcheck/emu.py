"""The host build of a kernel source: tests/host_emu/<name>.cpp compiled into a shared library, once per
session."""
import ctypes
import os
import subprocess

HOST_EMU = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "host_emu")
_built = {}


def build(tmp_path_factory, name):
    """ctypes.CDLL of host_emu/<name>.cpp.  -ffp-contract=off: no multiply-add is fused unless the source fuses it."""
    if name not in _built:
        out = str(tmp_path_factory.mktemp("emu") / f"lib{name}.so")
        subprocess.run(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-I", HOST_EMU, "-o", out,
                        os.path.join(HOST_EMU, name + ".cpp")], check=True)
        _built[name] = ctypes.CDLL(out)
    return _built[name]


def ptr(a):
    """The data pointer of a numpy array for a ctypes call; None passes NULL."""
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)
