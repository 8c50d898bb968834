"""Rebuilds MXNet NDArray-list checkpoints with the layout of the reference's shipped ones from tests/golden/checkpoints.npz
(make_golden_checkpoints.py): the same arrays in the same order, names and shapes; each array starts with the shipped
file's first values and continues with seeded noise."""
import os
import struct

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "checkpoints.npz")


def layout(kind):
    """(names, shapes, heads) of the shipped checkpoint `kind` ("s" or "cascade")."""
    d = np.load(GOLDEN)
    names, ndim, dims, head = d[f"{kind}_names"], d[f"{kind}_ndim"], d[f"{kind}_dims"], d[f"{kind}_head"]
    shapes, off = [], 0
    for n in ndim:
        shapes.append(tuple(int(x) for x in dims[off:off + n]))
        off += n
    return [str(x) for x in names], shapes, head


def write_checkpoint(path, kind, seed=0):
    """Writes the checkpoint and returns {gluon name: array} of what it holds."""
    names, shapes, head = layout(kind)
    rng = np.random.default_rng(seed)
    arrays = {}
    with open(path, "wb") as f:
        f.write(struct.pack("<QQQ", 0x112, 0, len(names)))
        for name, shape, h in zip(names, shapes, head):
            a = rng.standard_normal(int(np.prod(shape))).astype(np.float32)
            k = min(a.size, h.size)
            a[:k] = h[:k]
            a = a.reshape(shape)
            f.write(struct.pack("<IiI", 0xF993FAC9, 0, len(shape)))
            f.write(struct.pack(f"<{len(shape)}q", *shape))
            f.write(struct.pack("<iii", 1, 0, 0))      # cpu, device 0, float32
            f.write(a.tobytes())
            arrays[name] = a
        f.write(struct.pack("<Q", len(names)))
        for name in names:
            b = name.encode()
            f.write(struct.pack("<Q", len(b)) + b)
    return arrays
