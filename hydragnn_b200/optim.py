"""Flat-buffer optimizers: every optimizer ``hydragnn/utils/optimizer/optimizer.py`` selects, one sm_90a kernel per step.

``FlatOptimizer`` holds what they share: ONE flat fp32 buffer of parameters (the modules' parameters become views into it) and
one of gradients, the gradient gather after ``backward``, and the device vector {lr, grad_scale} the kernels read, so a
CUDA-graph-captured step follows a learning-rate scheduler and the 1/world gradient scale of the flat all-reduce is folded into
the update.  ``train_step``, ``GraphedTrainStep`` and ``PaddedGraphStep`` drive any of them through ``backward``, ``flat_g``,
``step(grad_scale)``, ``sync_hyper`` and ``state_tensors``.

``FlatSGD``, ``FlatAdam``, ``FlatAdamW``, ``FlatAdamax``, ``FlatAdagrad``, ``FlatAdadelta`` and ``FlatRMSprop`` are
``torch.optim.Optimizer``s with one param group: the group holds torch's keys with torch's defaults, the kernels follow
torch's single-tensor algorithms (AdamW's in fp32, see ``FlatAdamW``), and ``state_dict()`` / ``load_state_dict()`` speak the
matching ``torch.optim`` class's format, so optimizer checkpoints move between torch and the engine in both directions.  torch's
``maximize``, ``capturable``, ``differentiable``, ``foreach`` and ``fused`` flags, sparse gradients and more than one param
group are not supported.
"""
import torch

from . import ops

class FlatOptimizer(torch.optim.Optimizer):
    """Flat parameter / gradient buffers and the device hyperparameters shared by the flat optimizers.

    A subclass names ``torch_cls`` (the torch optimizer whose semantics and checkpoint format it has), ``hyper`` (the group keys
    it reads), ``buffer_keys()`` (torch's per-parameter state names under the current options, each one flat buffer here) and
    ``_update(group, state, grad_scale)`` (one kernel launch).  ``fixed`` holds the group values its kernel implements: a
    checkpoint whose group carries another value of one of these keys is refused, not run as a different algorithm.

    Only lr (and the gradient scale) reach a CUDA-graph-captured step through the device; the other hyperparameters are kernel
    arguments, fixed when the step is captured.  ``captured_hyper()`` names them: ``train`` re-captures its padded step when they
    differ from the captured ones; a hand-held ``GraphedTrainStep`` must be built again after changing them."""

    torch_cls = None
    hyper = ("lr",)
    has_step = True              # torch keeps a per-parameter "step" in the state (SGD does not)
    state_at_init = False        # torch creates the state at construction (Adagrad), not at the first step
    fixed = {"maximize": False, "differentiable": False, "decoupled_weight_decay": False}

    def __init__(self, model, defaults):
        name = type(self).__name__
        if isinstance(model, torch.nn.Module) and any(getattr(m, "graph_attr_modules_missing", lambda: False)() for m in model.modules()):
            # the buffer holds the parameters that exist now: a conditioning module created later would never be trained
            raise ValueError("%s: this model's graph-attribute conditioning modules are created at its first forward; run "
                             "one forward (or load the checkpoint) before building the optimizer" % name)
        params = [p for p in (model.parameters() if isinstance(model, torch.nn.Module) else model) if p.requires_grad]
        if self.torch_cls is not None:
            # torch validates the options and supplies the rest of its group keys (maximize, foreach, ...) with their defaults
            template = self.torch_cls([torch.zeros(1, requires_grad=True)], **defaults).param_groups[0]
            defaults = {k: v for k, v in template.items() if k != "params"}
        super().__init__(params, defaults)
        self.params = params
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        self.flat_p = torch.empty(n, dtype=torch.float32, device=dev)
        self.flat_g = torch.zeros(n, dtype=torch.float32, device=dev)
        off = 0
        self.slices = []
        for p in self.params:
            k = p.numel()
            self.flat_p[off:off + k].copy_(p.data.reshape(-1))
            p.data = self.flat_p[off:off + k].view_as(p.data)
            self.slices.append((off, k))
            off += k
        self.step_dev = torch.zeros(1, dtype=torch.float32, device=dev)
        lr = defaults["lr"]
        self.hyper_dev = torch.tensor([lr, 1.0], dtype=torch.float32, device=dev)      # {lr, grad_scale} read by the kernel
        self._hyper_host = (float(lr), 1.0)
        self.flat_state = {}
        self._alloc_state()

    @property
    def lr(self):
        return self.param_groups[0]["lr"]

    def zero_grad(self, set_to_none=True):
        for p in self.params:
            p.grad = None

    def backward(self, loss):
        """``loss.backward()`` with the weight-gradient kernels of leaf parameters left running on the side stream until the flat
        gradient is gathered (ops.deferred_weight_gradients), then ``gather_grads()``."""
        with ops.deferred_weight_gradients():
            loss.backward()
        return self.gather_grads()

    def gather_grads(self):
        """autograd's per-parameter gradients -> the flat buffer (parameters nobody used contribute zeros)."""
        ops.join_side_streams()                     # weight-gradient kernels run on a side stream (ops.fork_join)
        gs = [(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in self.params]
        torch.cat(gs, out=self.flat_g)
        return self.flat_g

    def sync_hyper(self, grad_scale=None):
        """Push lr / grad_scale to the device if they changed (a tiny async H2D copy, outside any captured graph)."""
        want = (float(self.param_groups[0]["lr"]), self._hyper_host[1] if grad_scale is None else float(grad_scale))
        if want != self._hyper_host:
            self.hyper_dev.copy_(torch.tensor(want, dtype=torch.float32), non_blocking=False)
            self._hyper_host = want

    def _sync_for_step(self, grad_scale):
        capturing = self.flat_p.is_cuda and torch.cuda.is_current_stream_capturing()
        if not capturing:
            self.sync_hyper(grad_scale)
        elif float(grad_scale) != self._hyper_host[1]:
            raise RuntimeError("%s: call sync_hyper(grad_scale) before capturing a step with a new gradient scale" % type(self).__name__)

    def step(self, grad_scale=1.0, closure=None):
        if not (self.flat_p.is_cuda and torch.cuda.is_current_stream_capturing()):
            self._alloc_state()             # momentum / amsgrad / centered may have been switched on through param_groups
        self._sync_for_step(grad_scale)
        self._update(self.param_groups[0], self.flat_state, grad_scale)

    def captured_hyper(self):
        """The hyperparameters a captured step holds as kernel arguments (every group key the update reads except lr)."""
        g = self.param_groups[0]
        return tuple(g[k] for k in self.hyper if k != "lr")

    # ---- state -----------------------------------------------------------------------------------------------------------
    def buffer_keys(self):
        """torch's per-parameter state names under the current options, in torch's order (one flat buffer each)."""
        return []

    def initial_value(self, key):
        return 0.0

    def state_tensors(self):
        """Every device tensor the update reads and writes besides the parameters, ``step_dev`` last: what a caller saves and
        restores around steps that must not count (the warm-up of a captured step)."""
        return [self.flat_state[k] for k in self.buffer_keys()] + [self.step_dev]

    def _alloc_state(self):
        """One zero-initialised (or ``initial_value``) flat buffer per state name the options need; buffers that exist are kept.
        A step captured before the set changed holds the old buffers: the padded fast path is dropped here so it re-captures."""
        keys = self.buffer_keys()
        if set(keys) == set(self.flat_state):
            return
        self.flat_state = {k: self.flat_state[k] if k in self.flat_state else torch.full_like(self.flat_p, self.initial_value(k))
                           for k in keys}
        self._hgb_fast = None

    # ---- the torch.optim checkpoint format ---------------------------------------------------------------------------------
    def state_dict(self):
        keys = self.buffer_keys()
        state = {}
        if (keys or self.has_step) and (self.state_at_init or float(self.step_dev) > 0):
            step = self.step_dev.detach().clone().reshape(()).cpu()
            for i, (off, k) in enumerate(self.slices):
                shp = self.params[i].shape
                st = {"step": step.clone()} if self.has_step else {}
                for key in keys:
                    st[key] = self.flat_state[key][off:off + k].view(shp).clone()
                state[i] = st
        group = {k: v for k, v in self.param_groups[0].items() if k != "params"}
        group["params"] = list(range(len(self.params)))
        return {"state": state, "param_groups": [group]}

    def load_state_dict(self, sd):
        name = type(self).__name__
        groups = sd["param_groups"]
        order = [i for g in groups for i in g["params"]]
        if len(order) != len(self.params):
            raise ValueError("%s.load_state_dict: %d parameters in the checkpoint, %d in the model" % (name, len(order), len(self.params)))
        g0 = groups[0]
        for key, value in self.fixed.items():
            if key in g0 and g0[key] != value:
                raise ValueError("%s.load_state_dict: the checkpoint's optimizer has %s=%s, which the flat step does not implement"
                                 % (name, key, g0[key]))
        for key in self.hyper:
            if key in g0:
                self.param_groups[0][key] = tuple(g0[key]) if isinstance(g0[key], list) else g0[key]
        self._alloc_state()                 # amsgrad / momentum / centered decide which buffers exist
        keys = self.buffer_keys()
        step, seen = None, False
        for j, (off, k) in zip(order, self.slices):
            st = sd["state"].get(j, sd["state"].get(str(j))) or {}
            for key in keys:
                if st.get(key) is not None:
                    self.flat_state[key][off:off + k].copy_(st[key].reshape(-1))
                    seen = True
                else:
                    self.flat_state[key][off:off + k].fill_(self.initial_value(key))
            if "step" in st:
                step = float(st["step"]) if step is None else max(step, float(st["step"]))
        if not self.has_step:               # SGD: a momentum buffer in the checkpoint means the first step has been taken
            step = 1.0 if seen else None
        self.step_dev.fill_(0.0 if step is None else step)
        self._hgb_fast = None               # a captured step holds the hyperparameters it was captured with


class FlatSGD(FlatOptimizer):
    """torch.optim.SGD over the flat buffers (``momentum_buffer`` when momentum != 0)."""
    torch_cls = torch.optim.SGD
    hyper = ("lr", "momentum", "dampening", "weight_decay", "nesterov")
    has_step = False

    def __init__(self, model, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False):
        super().__init__(model, dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov))

    def buffer_keys(self):
        return ["momentum_buffer"] if self.param_groups[0]["momentum"] != 0 else []

    def _update(self, g, s, grad_scale):
        ops.sgd_step(self.flat_p, self.flat_g, s.get("momentum_buffer"), self.step_dev, g["lr"], g["momentum"], g["dampening"],
                     g["nesterov"], g["weight_decay"], grad_scale, hyper_dev=self.hyper_dev)


class FlatAdam(FlatOptimizer):
    """torch.optim.Adam over the flat buffers (L2 weight decay added to the gradient; ``max_exp_avg_sq`` with amsgrad)."""
    torch_cls = torch.optim.Adam
    hyper = ("lr", "betas", "eps", "weight_decay", "amsgrad")

    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False):
        super().__init__(model, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad))

    def buffer_keys(self):
        return ["exp_avg", "exp_avg_sq"] + (["max_exp_avg_sq"] if self.param_groups[0]["amsgrad"] else [])

    def _update(self, g, s, grad_scale):
        ops.adam_step(self.flat_p, self.flat_g, s["exp_avg"], s["exp_avg_sq"], s.get("max_exp_avg_sq"), self.step_dev, g["lr"],
                      g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], g["amsgrad"], grad_scale, hyper_dev=self.hyper_dev)


class FlatAdamW(FlatOptimizer):
    """torch.optim.AdamW over the flat buffers (decoupled weight decay), the default of ``hydragnn/utils/optimizer/optimizer.py``.
    Its kernel takes fp32 hyperparameters and computes the bias corrections in fp32."""
    torch_cls = torch.optim.AdamW
    hyper = ("lr", "betas", "eps", "weight_decay")
    fixed = {**FlatOptimizer.fixed, "decoupled_weight_decay": True, "amsgrad": False}

    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2):
        super().__init__(model, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def buffer_keys(self):
        return ["exp_avg", "exp_avg_sq"]

    @property
    def m(self):
        """The flat first moment, ``flat_state["exp_avg"]``."""
        return self.flat_state["exp_avg"]

    @property
    def v(self):
        """The flat second moment, ``flat_state["exp_avg_sq"]``."""
        return self.flat_state["exp_avg_sq"]

    def _update(self, g, s, grad_scale):
        ops.adamw_step(self.flat_p, self.flat_g, s["exp_avg"], s["exp_avg_sq"], self.step_dev, g["lr"], g["betas"][0], g["betas"][1],
                       g["eps"], g["weight_decay"], grad_scale, hyper_dev=self.hyper_dev)


class FlatAdamax(FlatOptimizer):
    """torch.optim.Adamax over the flat buffers."""
    torch_cls = torch.optim.Adamax
    hyper = ("lr", "betas", "eps", "weight_decay")

    def __init__(self, model, lr=2e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        super().__init__(model, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))

    def buffer_keys(self):
        return ["exp_avg", "exp_inf"]

    def _update(self, g, s, grad_scale):
        ops.adamax_step(self.flat_p, self.flat_g, s["exp_avg"], s["exp_inf"], self.step_dev, g["lr"], g["betas"][0], g["betas"][1],
                        g["eps"], g["weight_decay"], grad_scale, hyper_dev=self.hyper_dev)


class FlatAdagrad(FlatOptimizer):
    """torch.optim.Adagrad over the flat buffers; like torch, the state (``sum`` = initial_accumulator_value) exists from
    construction on."""
    torch_cls = torch.optim.Adagrad
    hyper = ("lr", "lr_decay", "weight_decay", "initial_accumulator_value", "eps")
    state_at_init = True

    def __init__(self, model, lr=1e-2, lr_decay=0, weight_decay=0, initial_accumulator_value=0, eps=1e-10):
        super().__init__(model, dict(lr=lr, lr_decay=lr_decay, weight_decay=weight_decay,
                                     initial_accumulator_value=initial_accumulator_value, eps=eps))

    def buffer_keys(self):
        return ["sum"]

    def initial_value(self, key):
        return float(self.param_groups[0]["initial_accumulator_value"])

    def _update(self, g, s, grad_scale):
        ops.adagrad_step(self.flat_p, self.flat_g, s["sum"], self.step_dev, g["lr"], g["lr_decay"], g["weight_decay"], g["eps"],
                         grad_scale, hyper_dev=self.hyper_dev)


class FlatAdadelta(FlatOptimizer):
    """torch.optim.Adadelta over the flat buffers."""
    torch_cls = torch.optim.Adadelta
    hyper = ("lr", "rho", "eps", "weight_decay")

    def __init__(self, model, lr=1.0, rho=0.9, eps=1e-6, weight_decay=0):
        super().__init__(model, dict(lr=lr, rho=rho, eps=eps, weight_decay=weight_decay))

    def buffer_keys(self):
        return ["square_avg", "acc_delta"]

    def _update(self, g, s, grad_scale):
        ops.adadelta_step(self.flat_p, self.flat_g, s["square_avg"], s["acc_delta"], self.step_dev, g["lr"], g["rho"], g["eps"],
                          g["weight_decay"], grad_scale, hyper_dev=self.hyper_dev)


class FlatRMSprop(FlatOptimizer):
    """torch.optim.RMSprop over the flat buffers (``momentum_buffer`` when momentum > 0, ``grad_avg`` when centered)."""
    torch_cls = torch.optim.RMSprop
    hyper = ("lr", "alpha", "eps", "weight_decay", "momentum", "centered")

    def __init__(self, model, lr=1e-2, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False):
        super().__init__(model, dict(lr=lr, alpha=alpha, eps=eps, weight_decay=weight_decay, momentum=momentum, centered=centered))

    def buffer_keys(self):
        g = self.param_groups[0]
        return ["square_avg"] + (["momentum_buffer"] if g["momentum"] > 0 else []) + (["grad_avg"] if g["centered"] else [])

    def _update(self, g, s, grad_scale):
        ops.rmsprop_step(self.flat_p, self.flat_g, s["square_avg"], s.get("momentum_buffer"), s.get("grad_avg"), self.step_dev,
                         g["lr"], g["alpha"], g["eps"], g["weight_decay"], g["momentum"], g["centered"], grad_scale,
                         hyper_dev=self.hyper_dev)


def select_optimizer(model, config):
    """hydragnn/utils/optimizer/optimizer.py:select_optimizer on the engine: ``config["type"]`` names the optimizer and only
    ``config["learning_rate"]`` is passed, so every other hyperparameter takes torch's default, as in the reference.

    ``use_zero_redundancy`` builds the same flat optimizer: ZeRO shards only the optimizer state across ranks, not the
    arithmetic, and the engine's whole parameter set is a few MB, so every rank keeps the full state and computes the same
    update.  "FusedLAMB" (DeepSpeed's FusedLamb) is not implemented and is refused."""
    name = config["type"]
    if name == "FusedLAMB":
        raise ValueError("select_optimizer: the engine does not implement DeepSpeed's FusedLamb (\"FusedLAMB\"); choose SGD, Adam, "
                         "Adadelta, Adagrad, Adamax, AdamW or RMSprop")
    cls = {"SGD": FlatSGD, "Adam": FlatAdam, "Adadelta": FlatAdadelta, "Adagrad": FlatAdagrad, "Adamax": FlatAdamax,
           "AdamW": FlatAdamW, "RMSprop": FlatRMSprop}.get(name)
    if cls is None:
        raise NameError("The string used to identify the optimizer is NOT recognized")
    return cls(model, lr=config["learning_rate"])
