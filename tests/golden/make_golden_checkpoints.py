"""Generates tests/golden/checkpoints.npz: the layout of the reference's shipped checkpoints, small enough to commit.

    python tests/golden/make_golden_checkpoints.py <reference tree>

For weights/dbbSep30-1206_1000000.params (MaskFlownet-S) and weights/5adNov03-0005_1000000.params (MaskFlownet) it stores,
in file order, every array's gluon name, shape and the first HEAD values, and it stores the gluon parameter names that the
reference's own model file (network/MaskFlownet.py) gives MaskFlownet_S and MaskFlownet when constructed through the mx shim.
tests/test_host_logic.py rebuilds checkpoints of the same layout from this (tests/golden/ckpt.py) and runs the reader and
the name mapping on them, so the tests need neither the 42 / 83 MB files nor the reference tree.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HEAD = 64

CHECKPOINTS = {"s": "dbbSep30-1206_1000000.params", "cascade": "5adNov03-0005_1000000.params"}


def main(ref_dir):
    from maskflownet_b200 import mx, params
    from maskflownet_b200.mx import ndarray as F
    out = {}
    for key, fn in CHECKPOINTS.items():
        raw = params.read_params(os.path.join(ref_dir, "weights", fn))
        names = list(raw)
        shapes = [raw[k].shape for k in names]
        assert all(raw[k].dtype == np.float32 for k in names)
        out[f"{key}_names"] = np.array(names)
        out[f"{key}_ndim"] = np.array([len(s) for s in shapes], dtype=np.int64)
        out[f"{key}_dims"] = np.array([d for s in shapes for d in s], dtype=np.int64)
        out[f"{key}_head"] = np.stack([np.pad(raw[k].reshape(-1)[:HEAD], (0, max(0, HEAD - raw[k].size))) for k in names])
    ref = mx.load_reference_network(ref_dir)
    F.set_device("cpu")
    out["ref_s_param_names"] = np.array(sorted(ref.MaskFlownet_S(config=mx.Reader({})).collect_params()))
    out["ref_cascade_param_names"] = np.array(sorted(ref.MaskFlownet(config=mx.Reader({})).collect_params()))
    dst = os.path.join(ROOT, "tests", "golden", "checkpoints.npz")
    np.savez_compressed(dst, **out)
    print(dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
