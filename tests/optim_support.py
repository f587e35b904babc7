"""What the optimizer tests share: the option combinations every flat optimizer is checked over (every option of the table in
hydragnn_b200/optim.py's classes: momentum 0 and > 0, dampening, nesterov, weight decay 0 and > 0, amsgrad, lr_decay, the initial
accumulator, centered), the torch and flat classes by type name, the fp64 oracle trajectory and the hyperparameters as a kernel
receives them."""
import torch

import hydragnn_b200 as hb
from oracle import optim as oopt

FLAT = {"SGD": hb.FlatSGD, "Adam": hb.FlatAdam, "AdamW": hb.FlatAdamW, "Adamax": hb.FlatAdamax, "Adagrad": hb.FlatAdagrad,
        "Adadelta": hb.FlatAdadelta, "RMSprop": hb.FlatRMSprop}
TORCH = {n: getattr(torch.optim, n) for n in FLAT}

CASES = [
    ("SGD", dict(lr=0.05)),
    ("SGD", dict(lr=0.05, weight_decay=0.01)),
    ("SGD", dict(lr=0.05, momentum=0.9)),
    ("SGD", dict(lr=0.05, momentum=0.9, dampening=0.1, weight_decay=0.01)),
    ("SGD", dict(lr=0.05, momentum=0.9, nesterov=True, weight_decay=0.01)),
    ("Adam", dict(lr=0.01)),
    ("Adam", dict(lr=0.01, weight_decay=0.01)),
    ("Adam", dict(lr=0.01, amsgrad=True)),
    ("Adam", dict(lr=0.01, betas=(0.8, 0.99), amsgrad=True, weight_decay=0.01)),
    ("AdamW", dict(lr=0.01)),
    ("AdamW", dict(lr=0.01, betas=(0.8, 0.99), weight_decay=0.05)),
    ("Adamax", dict(lr=0.01)),
    ("Adamax", dict(lr=0.01, weight_decay=0.01, betas=(0.3, 0.9))),        # 1 - beta1 >= 0.5: lerp's other branch
    ("Adagrad", dict(lr=0.05)),
    ("Adagrad", dict(lr=0.05, lr_decay=0.05)),
    ("Adagrad", dict(lr=0.05, lr_decay=0.01, weight_decay=0.01, initial_accumulator_value=0.1)),
    ("Adadelta", dict(lr=1.0)),
    ("Adadelta", dict(lr=0.5, rho=0.8, weight_decay=0.01)),
    ("RMSprop", dict(lr=0.01)),
    ("RMSprop", dict(lr=0.01, momentum=0.9)),
    ("RMSprop", dict(lr=0.01, centered=True)),
    ("RMSprop", dict(lr=0.01, centered=True, momentum=0.5, weight_decay=0.01)),
]
IDS = ["%s-%s" % (n, "-".join("%s=%s" % kv for kv in sorted(hp.items()) if kv[0] != "lr") or "default") for n, hp in CASES]


def kernel_hp(name, hp):
    """``hp`` as the kernel receives it: hgb_adamw_step takes its betas, eps and weight decay as fp32."""
    if name != "AdamW":
        return hp
    h = {**oopt.DEFAULTS[name], **hp}
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))  # noqa: E731
    return {**h, "betas": tuple(f32(b) for b in h["betas"]), "eps": f32(h["eps"]), "weight_decay": f32(h["weight_decay"])}


def oracle_run(name, hp, p0, grads, lrs=None, grad_scale=1.0):
    """The fp64 oracle over ``grads`` (one per step) from ``p0``: (parameters, state) after the last step.  ``lrs``: the learning
    rate of every step (default: hp["lr"])."""
    p = p0.double().clone()
    st = oopt.new_state(name, p, **hp)
    for t, g in enumerate(grads, start=1):
        lr = hp["lr"] if lrs is None else lrs[t - 1]
        oopt.step(name, p, g.double() * grad_scale, st, t, **{**hp, "lr": lr})
    return p, st
