"""What the MACE distance-transform tests share: reading tests/golden/models_mace_transform.pt, whose state dicts and gradients
are stored packed by dtype (tests/golden/make_mace_transform_golden.py, ``pack``)."""
import torch


def unpack(packed):
    """The {name: tensor or None} dict ``pack`` stored, in its order."""
    out, offset = {}, {}
    for name, shape, dtype in zip(packed["names"], packed["shapes"], packed["dtypes"]):
        if shape is None:
            out[name] = None
            continue
        flat, o = packed["flat"][dtype], offset.get(dtype, 0)
        n = 1
        for s in shape:
            n *= s
        out[name] = flat[o:o + n].reshape(shape).clone()
        offset[dtype] = o + n
    return out


def load_golden(golden_dir):
    cases = torch.load(golden_dir + "/models_mace_transform.pt")
    for c in cases.values():
        c["state"], c["grads"] = unpack(c["state"]), unpack(c["grads"])
    return cases
