"""maskflownet_b200.mx -- a torch-backed stand-in for the slice of Apache MXNet that the reference's model files use.

The reference's hot path sits behind MXNet's operator namespace `F` (handed to HybridBlock.hybrid_forward) and the
gluon `nn` blocks (network/MaskFlownet.py:1-4, network/layer.py:1-6).  This package provides those names on torch CUDA
tensors so that `network/MaskFlownet.py` and `network/layer.py` import and run UNCHANGED:

    from maskflownet_b200 import mx
    ref = mx.load_reference_network("/path/to/MaskFlownet")     # registers the fake `mxnet`, imports network.MaskFlownet
    net = ref.MaskFlownet_S(config=mx.Reader({}))
    net.initialize(seed=0, device="cuda")
    preds, masks, srcs = net(mx.nd.array(img1), mx.nd.array(img2))

The four hot operators -- F.Correlation, F.contrib.DeformableConvolution, F.GridGenerator, F.BilinearSampler -- dispatch
to the hand-written sm_90a kernels through maskflownet_b200.ops (no fallback: they raise without a CUDA device).  The
remaining generic tensor helpers (concat, reshape codes, pad, Convolution/Deconvolution used by the reference's own
Upsample block, ...) map onto torch, which is the allocator/plumbing layer here.
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import types

from . import ndarray as nd  # noqa: F401
from . import gluon  # noqa: F401
from .ndarray import NDArray  # noqa: F401
from .config import Reader  # noqa: F401

symbol = nd  # hybrid_forward receives `F`; imperative and "symbolic" namespaces coincide here


class _Base(types.ModuleType):
    numeric_types = (float, int)


def install() -> types.ModuleType:
    """Register this package as `mxnet` (and its submodules) in sys.modules.  Idempotent; refuses to shadow a real MXNet."""
    existing = sys.modules.get("mxnet")
    if existing is not None and not getattr(existing, "__maskflow_shim__", False):
        raise RuntimeError("a real `mxnet` module is already imported; refusing to shadow it")
    me = sys.modules[__name__]
    me.__maskflow_shim__ = True
    base = _Base("mxnet.base")
    try:
        import numpy as _np
        base.numeric_types = (float, int, _np.generic)
    except Exception:  # pragma: no cover
        pass
    me.base = base
    me.ndarray = nd
    me.sym = nd
    sys.modules["mxnet"] = me
    sys.modules["mxnet.base"] = base
    sys.modules["mxnet.nd"] = nd
    sys.modules["mxnet.ndarray"] = nd
    sys.modules["mxnet.symbol"] = nd
    sys.modules["mxnet.gluon"] = gluon
    sys.modules["mxnet.gluon.nn"] = gluon.nn
    return me


def load_reference_network(repo_root: str):
    """Import <repo_root>/network/{layer,MaskFlownet}.py unchanged (without executing network/__init__.py, which pulls in
    the training pipeline).  Returns the imported `network.MaskFlownet` module."""
    install()
    net_dir = os.path.join(repo_root, "network")
    if not os.path.isfile(os.path.join(net_dir, "MaskFlownet.py")):
        raise FileNotFoundError(f"{net_dir}/MaskFlownet.py not found")
    pkg_name = "_mfn_reference_network"
    if pkg_name + ".MaskFlownet" in sys.modules:
        return sys.modules[pkg_name + ".MaskFlownet"]
    pkg = types.ModuleType(pkg_name)
    pkg.__path__ = [net_dir]
    sys.modules[pkg_name] = pkg
    for sub in ("layer", "MaskFlownet"):
        spec = importlib.util.spec_from_file_location(f"{pkg_name}.{sub}", os.path.join(net_dir, sub + ".py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[f"{pkg_name}.{sub}"] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, sub, mod)
    return sys.modules[pkg_name + ".MaskFlownet"]
