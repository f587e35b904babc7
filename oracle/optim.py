"""fp64 restatement of the seven update rules the flat optimizers implement, written from torch.optim's documented algorithms
(the single-tensor, ``foreach=False`` form; no maximize / capturable / differentiable): SGD, Adam, AdamW, Adamax, Adagrad,
Adadelta and RMSprop.

``step(name, p, g, state, t, **hp)`` updates the fp64 tensors ``p`` and ``state`` (a dict of torch's per-parameter state names)
in place for the 1-based step ``t`` and the hyperparameters ``hp`` (torch's keyword names, ``lr`` included).  ``new_state``
gives the state before the first step.  The gradient ``g`` is what the update sees (already scaled).
"""
import torch

DEFAULTS = {
    "SGD": dict(lr=1e-3, momentum=0.0, dampening=0.0, weight_decay=0.0, nesterov=False),
    "Adam": dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False),
    "AdamW": dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2),
    "Adamax": dict(lr=2e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0),
    "Adagrad": dict(lr=1e-2, lr_decay=0.0, weight_decay=0.0, initial_accumulator_value=0.0, eps=1e-10),
    "Adadelta": dict(lr=1.0, rho=0.9, eps=1e-6, weight_decay=0.0),
    "RMSprop": dict(lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0.0, momentum=0.0, centered=False),
}


def state_keys(name, **hp):
    hp = {**DEFAULTS[name], **hp}
    if name == "SGD":
        return ["momentum_buffer"] if hp["momentum"] != 0 else []
    if name in ("Adam", "AdamW"):
        return ["exp_avg", "exp_avg_sq"] + (["max_exp_avg_sq"] if hp.get("amsgrad") else [])
    if name == "RMSprop":
        return ["square_avg"] + (["momentum_buffer"] if hp["momentum"] > 0 else []) + (["grad_avg"] if hp["centered"] else [])
    return {"Adamax": ["exp_avg", "exp_inf"], "Adagrad": ["sum"], "Adadelta": ["square_avg", "acc_delta"]}[name]


def new_state(name, p, **hp):
    hp = {**DEFAULTS[name], **hp}
    init = hp["initial_accumulator_value"] if name == "Adagrad" else 0.0
    return {k: torch.full_like(p, float(init)) for k in state_keys(name, **hp)}


def step(name, p, g, state, t, **hp):
    hp = {**DEFAULTS[name], **hp}
    lr, wd = hp["lr"], hp["weight_decay"]
    if name == "AdamW":                           # decoupled decay of the parameters
        p.mul_(1 - lr * wd)
    elif wd != 0:                                 # every other one adds L2 decay to the gradient
        g = g + wd * p
    if name == "SGD":
        mom = hp["momentum"]
        if mom != 0:
            buf = state["momentum_buffer"]
            if t == 1:
                buf.copy_(g)                      # the first step takes the gradient as it is
            else:
                buf.mul_(mom).add_((1 - hp["dampening"]) * g)
            g = g + mom * buf if hp["nesterov"] else buf
        p.sub_(lr * g)
    elif name in ("Adam", "AdamW"):
        b1, b2 = hp["betas"]
        m, v = state["exp_avg"], state["exp_avg_sq"]
        m.mul_(b1).add_((1 - b1) * g)
        v.mul_(b2).add_((1 - b2) * g * g)
        if hp.get("amsgrad"):
            torch.maximum(state["max_exp_avg_sq"], v, out=state["max_exp_avg_sq"])
            v = state["max_exp_avg_sq"]
        bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
        p.sub_(lr / bc1 * m / (v.sqrt() / bc2 ** 0.5 + hp["eps"]))
    elif name == "Adamax":
        b1, b2 = hp["betas"]
        m, u = state["exp_avg"], state["exp_inf"]
        m.mul_(b1).add_((1 - b1) * g)
        torch.maximum(u * b2, g.abs() + hp["eps"], out=u)
        p.sub_(lr / (1 - b1 ** t) * m / u)
    elif name == "Adagrad":
        s = state["sum"]
        s.add_(g * g)
        clr = lr / (1 + (t - 1) * hp["lr_decay"])
        p.sub_(clr * g / (s.sqrt() + hp["eps"]))
    elif name == "Adadelta":
        rho, eps = hp["rho"], hp["eps"]
        sq, acc = state["square_avg"], state["acc_delta"]
        sq.mul_(rho).add_((1 - rho) * g * g)
        delta = (acc + eps).sqrt() / (sq + eps).sqrt() * g
        acc.mul_(rho).add_((1 - rho) * delta * delta)
        p.sub_(lr * delta)
    elif name == "RMSprop":
        a, eps, mom = hp["alpha"], hp["eps"], hp["momentum"]
        sq = state["square_avg"]
        sq.mul_(a).add_((1 - a) * g * g)
        if hp["centered"]:
            ga = state["grad_avg"]
            ga.mul_(a).add_((1 - a) * g)
            avg = (sq - ga * ga).sqrt() + eps
        else:
            avg = sq.sqrt() + eps
        if mom > 0:
            buf = state["momentum_buffer"]
            buf.mul_(mom).add_(g / avg)
            p.sub_(lr * buf)
        else:
            p.sub_(lr * g / avg)
    else:
        raise NameError("oracle.optim: unknown optimizer %r" % name)
    return p, state
