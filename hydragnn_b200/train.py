"""Data-parallel training step of the engine.

Mirror of the hot loop ``train()`` in hydragnn/train/train_validate_test.py:629-801 and of the DDP wrap in
hydragnn/utils/distributed/distributed.py:396-481, redesigned for one NVSwitch box:

* parameters and gradients live in ONE flat fp32 buffer each (the modules hold views), so the optimizer (a
  ``FlatOptimizer`` of optim.py, AdamW by default) is a single fused kernel and the only collective of the step is ONE
  ``all_reduce`` over the flat gradient (graphs shard by rank with no other communication -- SURVEY 8e); the 1/world_size
  scaling is folded into the optimizer kernel;
* no mpi4py anywhere on the step path (the reference's per-epoch ``MPI.allreduce(nbatch, MIN)``,
  :672, becomes a ``dist.all_reduce(MIN)``);
* ``GraphedTrainStep`` captures forward + loss + backward + flatten + optimizer of a fixed-shape batch in a CUDA
  graph (all kernels are launched through ctypes on the capturing stream; nothing synchronises).
"""
import torch
import torch.distributed as dist

from . import ops
from .optim import FlatOptimizer
from .stacks import forget_plans

PRECISION_MAP = {"bf16": torch.float32, "fp32": torch.float32}     # parameters stay fp32 (reference :43-49)


def resolve_precision(precision):
    prec = {"bfloat16": "bf16", "float32": "fp32", "float": "fp32", None: "fp32"}.get(precision, precision)
    prec = str(prec).lower()
    if prec in ("fp64", "float64", "double"):
        raise ValueError("Unsupported precision fp64: the b200 engine computes in fp32 / bf16")
    if prec not in PRECISION_MAP:
        raise ValueError("Unsupported precision %s. Choose from %s." % (precision, list(PRECISION_MAP)))
    return prec, PRECISION_MAP[prec], (torch.bfloat16 if prec == "bf16" else None)


def move_batch_to_device(data, param_dtype=torch.float32, device=None):
    """hydragnn/train/train_validate_test.py:74-84: cast floats, move everything."""
    for key, value in data.items():
        if torch.is_tensor(value) and torch.is_floating_point(value):
            data[key] = value.to(dtype=param_dtype)
    return data.to(device, non_blocking=True)


def get_head_indices(model, data):
    """Single-head / all-graph-head cases of hydragnn/train/train_validate_test.py:494-557."""
    m = getattr(model, "module", model)
    if m.num_heads == 1:
        return [torch.arange(data.y.shape[0], device=data.y.device)]
    if all(t == "graph" for t in m.head_type):
        dims, tot = m.head_dims, sum(m.head_dims)
        g = data.num_graphs
        base = torch.arange(g, device=data.y.device) * tot
        out, off = [], 0
        for d in dims:
            out.append((base[:, None] + off + torch.arange(d, device=data.y.device)[None, :]).reshape(-1))
            off += d
        return out
    y_loc = data.y_loc.to(data.y.device)
    start = (torch.cumsum(y_loc[:, -1], 0) - y_loc[:, -1]).view(-1, 1)
    out = []
    for ih in range(m.num_heads):
        lo, hi = (start + y_loc[:, ih:ih + 1]).flatten().tolist(), (start + y_loc[:, ih + 1:ih + 2]).flatten().tolist()
        out.append(torch.cat([torch.arange(a, b, device=data.y.device) for a, b in zip(lo, hi)]))
    return out


class DistributedModel(torch.nn.Module):
    """Stand-in for the DDP wrapper: ``.module`` is the model; gradient averaging is done on the flat buffer
    by ``train_step`` (one all-reduce), not by per-bucket hooks."""

    def __init__(self, module):
        super().__init__()
        self.module = module

    def forward(self, data):
        return self.module(data)


def get_distributed_model(model, verbosity=0, **_):
    if dist.is_initialized():
        # same starting point on every rank (DDP broadcasts rank 0's parameters at wrap time)
        for p in model.parameters():
            dist.broadcast(p.data, src=0)
    return DistributedModel(model)


def world():
    return (dist.get_world_size(), dist.get_rank()) if dist.is_initialized() else (1, 0)


def train_step(model, opt, data, compute_grad_energy=False, head_index=None):
    """forward -> loss -> backward -> flat all-reduce -> fused flat optimizer step.  Returns (loss, tasks_loss)
    (hydragnn/train/train_validate_test.py:702-769 without the tracing scaffolding)."""
    m = model.module
    opt.zero_grad()
    if compute_grad_energy:
        data.pos.requires_grad_(True)
        pred = model(data)
        loss, tasks = m.energy_force_loss(pred, data)
    else:
        if head_index is None:
            head_index = get_head_indices(model, data)
        pred = model(data)
        loss, tasks = m.loss(pred, data.y, head_index)
    flat = opt.backward(loss)
    ws, _ = world()
    if ws > 1:
        dist.all_reduce(flat)                                       # the only collective of the step
    opt.step(grad_scale=1.0 / ws)
    return loss.detach(), [t.detach() for t in tasks]


def _capturable_allreduce(flat):
    """The step's only collective, on the CURRENT stream (NCCL collectives are CUDA-graph capturable)."""
    dist.all_reduce(flat)


class GraphedTrainStep:
    """CUDA-graph capture of ``train_step`` for a fixed-shape batch living in static device buffers: forward + loss + backward
    + flatten + the flat NCCL all-reduce + fused AdamW are ONE graph (`hydragnn/utils/distributed/distributed.py:479` and
    `train_validate_test.py:737-769` in one replay).  ``refill(data)`` copies a new batch of the same shape -- positions,
    features, targets AND topology (``edge_index`` / ``batch``) -- into the static buffers; the index plans (CSR views of
    ``edge_index``, graph offsets) are rebuilt INSIDE the captured region, so a refilled topology is honoured.  With
    ``neighbour_build=(radius, max_neighbours)`` the radius graph itself is part of the captured step (edge count promised by the
    warm-up run and verified on the device -- ``ops.check_guard``)."""

    def __init__(self, model, opt, static_data, compute_grad_energy=False, warmup=3, capture_allreduce=True):
        self.model, self.opt, self.data, self.mlip = model, opt, static_data, compute_grad_energy
        self.head_index = None if compute_grad_energy else get_head_indices(model, static_data)
        self.ws, _ = world()
        self.capture_allreduce = bool(capture_allreduce)
        self.opt.sync_hyper(1.0 / self.ws)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._fwd_bwd()
                if self.ws > 1:
                    dist.all_reduce(self.opt.flat_g)
                self.opt.step(1.0 / self.ws)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.g_opt = None
        self.g_fb = torch.cuda.CUDAGraph()
        one_graph = self.ws == 1 or self.capture_allreduce
        with ops.capture_graph(self.g_fb):
            self._fwd_bwd()
            if one_graph:
                if self.ws > 1:
                    _capturable_allreduce(self.opt.flat_g)
                self.opt.step(1.0 / self.ws)
        if not one_graph:
            self.g_opt = torch.cuda.CUDAGraph()
            with ops.capture_graph(self.g_opt):
                self.opt.step(1.0 / self.ws)

    def _fwd_bwd(self):
        m = self.model.module
        d = self.data
        forget_plans(d)                     # index plans are part of the step: a refill may bring new edges and elements
        self.opt.zero_grad()
        if self.mlip:
            d.pos.requires_grad_(True)
            pred = self.model(d)
            loss, _ = m.energy_force_loss(pred, d)
        else:
            pred = self.model(d)
            loss, _ = m.loss(pred, d.y, self.head_index)
        self.opt.backward(loss)
        self.loss = loss.detach()

    def refill(self, data):
        for k, v in data.items():
            if torch.is_tensor(v):
                dst = self.data[k]
                if dst.shape != v.shape:
                    raise ValueError("GraphedTrainStep.refill: %s has shape %s, the captured step has %s" % (k, tuple(v.shape), tuple(dst.shape)))
                dst.detach().copy_(v, non_blocking=True)

    def run(self):
        self.opt.sync_hyper()                       # a scheduler may have changed the learning rate
        self.g_fb.replay()
        if self.g_opt is not None:
            dist.all_reduce(self.opt.flat_g)
            self.g_opt.replay()
        return self.loss


def _train_fast(loader, model, opt, compute_grad_energy, neighbour_build):
    """The epoch through ONE capacity-padded captured step (hydragnn_b200/padded.py): no per-step host synchronisation; the
    epoch sums stay on the device until the end."""
    from .padded import PaddedGraphStep
    dev = next(model.parameters()).device
    nbatch = len(loader)
    if dist.is_initialized():
        t = torch.tensor([nbatch], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        nbatch = int(t)
    fast = getattr(opt, "_hgb_fast", None)
    total = tasks_tot = None
    nsamp = 0
    for ibatch, data in enumerate(loader):
        if ibatch >= nbatch:
            break
        if (fast is None or fast.model is not model or fast.mlip != bool(compute_grad_energy) or fast.nb != neighbour_build
                or fast.hyper != opt.captured_hyper()):             # hyperparameters other than lr are fixed at capture
            fast = opt._hgb_fast = PaddedGraphStep(model, opt, data, compute_grad_energy, neighbour_build)
        g = fast.load(data)
        loss, tasks = fast.run()
        total = loss * g if total is None else total + loss * g
        tasks_tot = tasks * g if tasks_tot is None else tasks_tot + tasks * g
        nsamp += g
    fast.check()                                              # one host read per epoch: device guards of the captured steps
    return total / nsamp, tasks_tot / nsamp


def train(loader, model, opt, verbosity=0, profiler=None, use_deepspeed=False, compute_grad_energy=False, precision="fp32",
          fast=None, neighbour_build=None):
    """Epoch loop with the reference's signature and return values (train_error, tasks_error).

    ``fast`` (default: on for models ``padded.supported`` accepts): run every batch through one capacity-padded CUDA-graph step
    instead of eager launches -- same arithmetic, no per-step host sync.  ``neighbour_build`` = (radius, max_neighbours) builds
    the radius graph on the device inside that step; by default the batches carry ``edge_index`` as the reference's do."""
    resolve_precision(precision)
    dev = next(model.parameters()).device
    from . import padded
    if fast is None:
        fast = dev.type == "cuda" and padded.supported(model) and isinstance(opt, FlatOptimizer)
    if fast:
        model.train()
        train_error, tasks_error = _train_fast(loader, model, opt, compute_grad_energy, neighbour_build)
        ws, _ = world()
        if ws > 1:
            dist.all_reduce(train_error)
            dist.all_reduce(tasks_error)
            train_error, tasks_error = train_error / ws, tasks_error / ws
        return train_error, tasks_error
    total, tasks_tot, nsamp = None, None, 0
    model.train()
    nbatch = len(loader)
    if dist.is_initialized():
        t = torch.tensor([nbatch], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        nbatch = int(t)
    for ibatch, data in enumerate(loader):
        if ibatch >= nbatch:
            break
        data = move_batch_to_device(data, torch.float32, dev)
        loss, tasks = train_step(model, opt, data, compute_grad_energy)
        g = data.num_graphs
        total = loss * g if total is None else total + loss * g
        tl = torch.stack(tasks) * g
        tasks_tot = tl if tasks_tot is None else tasks_tot + tl
        nsamp += g
    train_error, tasks_error = total / nsamp, tasks_tot / nsamp
    ws, _ = world()
    if ws > 1:
        dist.all_reduce(train_error)
        dist.all_reduce(tasks_error)
        train_error, tasks_error = train_error / ws, tasks_error / ws
    return train_error, tasks_error


@torch.no_grad()
def _eval_no_force(model, data, head_index):
    pred = model(data)
    return model.module.loss(pred, data.y, head_index), pred


def validate(loader, model, verbosity=0, reduce_ranks=True, compute_grad_energy=False, precision="fp32"):
    """hydragnn/train/train_validate_test.py:805-873 (losses only)."""
    dev = next(model.parameters()).device
    model.eval()
    total, tasks_tot, nsamp = None, None, 0
    for data in loader:
        data = move_batch_to_device(data, torch.float32, dev)
        if compute_grad_energy:
            with torch.enable_grad():
                data.pos.requires_grad_(True)
                pred = model(data)
                loss, tasks = model.module.energy_force_loss(pred, data, create_graph=False)
            loss, tasks = loss.detach(), [t.detach() for t in tasks]
        else:
            (loss, tasks), _ = _eval_no_force(model, data, get_head_indices(model, data))
        g = data.num_graphs
        total = loss * g if total is None else total + loss * g
        tl = torch.stack(tasks) * g
        tasks_tot = tl if tasks_tot is None else tasks_tot + tl
        nsamp += g
    err, terr = total / nsamp, tasks_tot / nsamp
    ws, _ = world()
    if reduce_ranks and ws > 1:
        dist.all_reduce(err)
        dist.all_reduce(terr)
        err, terr = err / ws, terr / ws
    return err, terr
