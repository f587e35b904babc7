"""Generate tests/golden/optimizers.pt by running the REFERENCE's own ``select_standard_optimizer``
(hydragnn/utils/optimizer/optimizer.py), AST-extracted because its module imports hydragnn.utils.distributed and DeepSpeed at top
level; ``get_device_name`` is stubbed ("cpu") and DeepSpeed is absent.  Run in the build container only.

    python tests/golden/make_optimizer_golden.py      # writes optimizers.pt, nothing else

For each of the seven types the reference selects (SGD, Adam, Adadelta, Adagrad, Adamax, AdamW, RMSprop), built with
learning_rate 0.01 on a fixed fp64 parameter set, the golden holds

* ``class``: the torch.optim class name the reference builds, ``group``: its param group without ``params``;
* ``params0`` and ``grads`` (one gradient list per step) and, after every one of ``STEPS`` steps, the parameters and the
  per-parameter state (``trajectory``: a list of {"params": [...], "state": [{name: tensor}, ...]}).

``errors["unknown"]`` holds what the reference raises for an unknown type.
"""
import os
import sys

import torch

from record import REF, refusal, save

HERE = os.path.dirname(os.path.abspath(__file__))
TYPES = ("SGD", "Adam", "Adadelta", "Adagrad", "Adamax", "AdamW", "RMSprop")
STEPS = 4
LR = 0.01


def reference_select():
    import make_golden as mg
    glb = {"torch": torch, "get_device_name": lambda *a, **k: "cpu", "deepspeed_available": False}
    mg._extract(REF + "/hydragnn/utils/optimizer/optimizer.py", ["select_standard_optimizer"], glb)
    return glb["select_standard_optimizer"]


def main():
    select = reference_select()
    gen = torch.Generator().manual_seed(2024)
    shapes = [(3, 4), (4,), (2, 2, 3)]
    params0 = [torch.randn(s, generator=gen, dtype=torch.float64) for s in shapes]
    grads = [[torch.randn(s, generator=gen, dtype=torch.float64) for s in shapes] for _ in range(STEPS)]
    out = {"params0": params0, "grads": grads, "lr": LR, "types": {}, "errors": {}}
    for t in TYPES:
        model = torch.nn.ParameterList([torch.nn.Parameter(p.clone()) for p in params0])
        opt = select(model, {"type": t, "learning_rate": LR})
        group = {k: v for k, v in opt.param_groups[0].items() if k != "params"}
        traj = []
        for step in range(STEPS):
            for p, g in zip(model, grads[step]):
                p.grad = g.clone()
            opt.step()
            traj.append({"params": [p.detach().clone() for p in model],
                         "state": [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in opt.state[p].items()} for p in model]})
        out["types"][t] = {"class": type(opt).__name__, "group": group, "trajectory": traj}
    model = torch.nn.ParameterList([torch.nn.Parameter(p.clone()) for p in params0])
    out["errors"]["unknown"] = refusal(lambda: select(model, {"type": "Lion", "learning_rate": LR}))
    save(out, os.path.join(HERE, "optimizers.pt"))


if __name__ == "__main__":
    sys.exit(main())
