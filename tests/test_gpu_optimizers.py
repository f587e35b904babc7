"""The flat optimizer steps on the GPU: every kernel (hgb_optim_flat.cu) against the fp64 oracle (oracle/optim.py) and against
torch.optim in fp32 on the GPU, over every option combination of optim_support.CASES, sizes 0 .. 1 000 003 and grad_scale 1 and
0.25; a CUDA-graph-captured step following a learning rate changed between replays; torch <-> flat checkpoints on the GPU;
training through hb.train on the captured and the eager path against the same loop driven by torch.optim; FlatAdamW's captured
step bit for bit the kernel call it always made.

Tolerance of the kernel checks: fp32 elementwise arithmetic against fp64, max |flat - ref| <= 1e-5 * max |ref| for the parameters
and every state tensor after 10 steps, on gradients whose magnitudes are bounded away from zero (see the kernel test); AdamW's
exp_avg_sq against torch's: 2e-5, for the fp32 betas its kernel takes."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import ops  # noqa: E402
from hydragnn_b200.synthetic import ARCH, WORKLOADS  # noqa: E402
from optim_support import CASES, FLAT, IDS, TORCH, kernel_hp, oracle_run  # noqa: E402
from oracle import optim as oopt  # noqa: E402
from stack_support import _loader  # noqa: E402

DEV = "cuda"
RTOL = 1e-5
STEPS = 10


def _close(a, ref, rtol=RTOL):
    a, ref = a.double(), ref.double()
    err = float((a - ref).abs().max()) if a.numel() else 0.0
    scale = float(ref.abs().max()) if ref.numel() else 0.0
    assert err <= rtol * scale + 1e-30, (err, scale)


def _launch(name, hp, p, g, st, step_dev, grad_scale):
    """One flat step through the ops wrapper with state dict ``st`` (torch's names)."""
    h = {**oopt.DEFAULTS[name], **hp}
    if name == "SGD":
        ops.sgd_step(p, g, st.get("momentum_buffer"), step_dev, h["lr"], h["momentum"], h["dampening"], h["nesterov"],
                     h["weight_decay"], grad_scale)
    elif name == "Adam":
        ops.adam_step(p, g, st["exp_avg"], st["exp_avg_sq"], st.get("max_exp_avg_sq"), step_dev, h["lr"], h["betas"][0],
                      h["betas"][1], h["eps"], h["weight_decay"], h["amsgrad"], grad_scale)
    elif name == "AdamW":
        ops.adamw_step(p, g, st["exp_avg"], st["exp_avg_sq"], step_dev, h["lr"], h["betas"][0], h["betas"][1], h["eps"],
                       h["weight_decay"], grad_scale)
    elif name == "Adamax":
        ops.adamax_step(p, g, st["exp_avg"], st["exp_inf"], step_dev, h["lr"], h["betas"][0], h["betas"][1], h["eps"],
                        h["weight_decay"], grad_scale)
    elif name == "Adagrad":
        ops.adagrad_step(p, g, st["sum"], step_dev, h["lr"], h["lr_decay"], h["weight_decay"], h["eps"], grad_scale)
    elif name == "Adadelta":
        ops.adadelta_step(p, g, st["square_avg"], st["acc_delta"], step_dev, h["lr"], h["rho"], h["eps"], h["weight_decay"],
                          grad_scale)
    else:
        ops.rmsprop_step(p, g, st["square_avg"], st.get("momentum_buffer"), st.get("grad_avg"), step_dev, h["lr"], h["alpha"],
                         h["eps"], h["weight_decay"], h["momentum"], h["centered"], grad_scale)


@pytest.mark.parametrize("grad_scale", [1.0, 0.25])
@pytest.mark.parametrize("count", [0, 1, 3, 31, 4097, 1_000_003])
@pytest.mark.parametrize("name,hp", CASES, ids=IDS)
def test_kernel_matches_fp64_oracle_and_torch(name, hp, count, grad_scale):
    gen = torch.Generator(device=DEV).manual_seed(count + 7)
    p0 = torch.randn(count, device=DEV, generator=gen)
    # |g| in [0.5, 1.5): the scaled gradient stays clear of the weight-decay term, so no decayed gradient sits at its own rounding
    # level -- there the normalising rules (RMSprop, Adam, ... whose first step is about lr * sign(g)) are ill-conditioned in any
    # fp32 implementation, torch's included
    grads = [(torch.rand(count, device=DEV, generator=gen) + 0.5) * torch.randn(count, device=DEV, generator=gen).sign()
             for _ in range(STEPS)]
    p = p0.clone()
    st = {k: v.float() for k, v in oopt.new_state(name, p0.double(), **hp).items()}
    step_dev = torch.zeros(1, device=DEV)
    for g in grads:
        _launch(name, hp, p, g, st, step_dev, grad_scale)
    assert float(step_dev) == STEPS
    po, so = oracle_run(name, kernel_hp(name, hp), p0, grads, grad_scale=grad_scale)
    _close(p, po)
    for k in so:
        _close(st[k], so[k])
    # torch.optim in fp32 on the GPU, single-tensor path
    q = torch.nn.Parameter(p0.clone())
    opt = TORCH[name]([q], foreach=False, **hp)
    for g in grads:
        q.grad = g * grad_scale
        opt.step()
    _close(p, q.detach())
    for k in so:
        # AdamW's kernel takes fp32 betas: its 1.f - 0.999f is 1.29e-5 relative from torch's float(1 - 0.999) (the offset
        # test_adamw_distance_to_torch pins), and exp_avg_sq carries that offset
        _close(st[k], opt.state[q][k], rtol=2e-5 if (name, k) == ("AdamW", "exp_avg_sq") else RTOL)


def _toy(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(7, 33), torch.nn.Linear(33, 5)).to(DEV)


@pytest.mark.parametrize("name,hp", CASES, ids=IDS)
def test_captured_step_follows_the_learning_rate_between_replays(name, hp):
    """One step() captured in a CUDA graph, replayed 5 times with the lr changed through param_groups between replays (and a
    new gradient each time), equals 5 eager steps bit for bit -- SGD's first-step copy and Adagrad's decayed lr included."""
    gen = torch.Generator(device=DEV).manual_seed(1)
    ma, mb = _toy(), _toy()
    oa, ob = FLAT[name](ma, **hp), FLAT[name](mb, **hp)
    grads = [torch.randn(oa.flat_g.shape, device=DEV, generator=gen) for _ in range(5)]
    lrs = [hp["lr"] * f for f in (1.0, 0.5, 0.5, 0.2, 0.05)]
    warm = FLAT[name](_toy(), **hp)                    # loads the kernels outside the capture
    warm.step()
    oa.sync_hyper(1.0)
    graph = torch.cuda.CUDAGraph()
    with ops.capture_graph(graph):
        oa.step()
    for t in range(5):
        oa.param_groups[0]["lr"] = lrs[t]
        ob.param_groups[0]["lr"] = lrs[t]
        oa.flat_g.copy_(grads[t])
        ob.flat_g.copy_(grads[t])
        oa.sync_hyper()
        graph.replay()
        ob.step()
    torch.cuda.synchronize()
    assert torch.equal(oa.flat_p, ob.flat_p)
    for x, y in zip(oa.state_tensors(), ob.state_tensors()):
        assert torch.equal(x, y)
    assert float(oa.step_dev) == 5.0


@pytest.mark.parametrize("name,hp", CASES, ids=IDS)
def test_checkpoints_both_ways_on_the_gpu(name, hp):
    """torch.optim.X steps 3 times; FlatX loads its checkpoint and steps 3 times; torch.optim.X loads FlatX's checkpoint and steps
    twice more.  Every leg agrees with torch stepping throughout."""
    gen = torch.Generator(device=DEV).manual_seed(2)
    shapes = [p.shape for p in _toy().parameters()]
    grads = [[torch.randn(s, device=DEV, generator=gen) for s in shapes] for _ in range(8)]

    def torch_steps(model, opt, steps):
        for s in steps:
            for p, g in zip(model.parameters(), grads[s]):
                p.grad = g.clone()
            opt.step()

    ref_m = _toy()
    torch_steps(ref_m, TORCH[name](ref_m.parameters(), foreach=False, **hp), range(8))
    a = _toy()
    oa = TORCH[name](a.parameters(), foreach=False, **hp)
    torch_steps(a, oa, range(3))
    b = _toy()
    b.load_state_dict(a.state_dict())
    ob = FLAT[name](b, lr=123.0)
    ob.load_state_dict(oa.state_dict())
    for s in range(3, 6):
        for p, g in zip(b.parameters(), grads[s]):
            p.grad = g.clone()
        ob.gather_grads()
        ob.step()
    mid = _toy()
    torch_steps(mid, TORCH[name](mid.parameters(), foreach=False, **hp), range(6))
    for p, q in zip(b.parameters(), mid.parameters()):
        _close(p.detach(), q.detach())
    c = _toy()
    c.load_state_dict(b.state_dict())
    oc = TORCH[name](c.parameters(), lr=123.0, foreach=False)
    oc.load_state_dict(ob.state_dict())
    torch_steps(c, oc, range(6, 8))
    for p, q in zip(c.parameters(), ref_m.parameters()):
        _close(p.detach(), q.detach())


TRAIN_CASES = [("qm9_painn", False, False), ("qm9_painn", False, True), ("md17_egnn", True, False), ("md17_egnn", True, True),
               ("lj_egnn", True, False)]


def _torch_epoch(loader, model, opt, mlip):
    """The eager epoch of hb.train driven by torch.optim (per-parameter gradients, torch's own step): (train_error, tasks_error),
    the graph-weighted means hb.train returns."""
    from hydragnn_b200.train import move_batch_to_device
    m = model.module
    model.train()
    total, tasks_tot, nsamp = 0.0, 0.0, 0
    for b in loader:
        data = move_batch_to_device(b, torch.float32, DEV)
        opt.zero_grad(set_to_none=True)
        if mlip:
            data.pos.requires_grad_(True)
            loss, tasks = m.energy_force_loss(model(data), data)
        else:
            loss, tasks = m.loss(model(data), data.y, hb.get_head_indices(model, data))
        loss.backward()
        ops.join_side_streams()
        opt.step()
        g = data.num_graphs
        total = total + loss.detach() * g
        tasks_tot = tasks_tot + torch.stack([t.detach() for t in tasks]) * g
        nsamp += g
    return total / nsamp, tasks_tot / nsamp


def _flat_params(model):
    return torch.cat([p.detach().reshape(-1) for p in model.parameters()])


def _displacement_rel(p, q, p0):
    """rel-L2 of the distance travelled: |(p - p0) - (q - p0)| / |q - p0|.  Scale-free, so it judges Adadelta's and SGD's small
    moves as strictly as Adam's: leaving out or repeating one of the ten updates changes it by about 0.1, skipping them all by 1."""
    d = q - p0
    assert float(d.norm()) > 0.0
    return float((p - q).norm() / d.norm())


DISPLACEMENT_RTOL = 1e-2


@pytest.mark.parametrize("opt_type", list(FLAT))
@pytest.mark.parametrize("name,mlip,build", TRAIN_CASES)
def test_train_fast_path_equals_eager_and_torch(name, mlip, build, opt_type):
    """hb.train with select_optimizer's optimizer over two epochs (ten steps) of batches whose graph / node / edge counts all
    differ: the captured padded step, the eager path and the same loop driven by torch.optim give the same per-epoch losses (the
    tolerances of test_gpu_round2's AdamW check) and the same parameter displacement.

    The displacement is compared as one vector (``_displacement_rel`` <= 1e-2), not weight by weight: the normalising rules move
    a weight whose gradient sits at rounding level by about lr * sign(g) (RMSprop: 10 lr on its first step), so a handful of such
    weights differ between any two fp32 gradient paths while the trajectory as a whole agrees to ~1e-3."""
    w = WORKLOADS[name]
    loader = _loader(name, [24, 17, 31, 24, 9], with_edges=True)
    nb = (w["radius"], w["max_neighbours"]) if build else None
    m1 = hb.get_distributed_model(hb.create_model(**ARCH[name]))
    m2, m3 = copy.deepcopy(m1), copy.deepcopy(m1)
    p0 = _flat_params(m1).clone()
    cfg = {"type": opt_type, "learning_rate": 1e-3}
    o1 = hb.select_optimizer(m1, cfg)
    o2 = hb.select_optimizer(m2, dict(cfg, use_zero_redundancy=True))
    o3 = TORCH[opt_type](m3.parameters(), lr=1e-3, foreach=False)
    for epoch in range(2):
        e_fast, t_fast = hb.train([b.clone() for b in loader], m1, o1, compute_grad_energy=mlip, neighbour_build=nb)
        e_eager, t_eager = hb.train([b.clone() for b in loader], m2, o2, compute_grad_energy=mlip, fast=False)
        e_torch, t_torch = _torch_epoch([b.clone() for b in loader], m3, o3, mlip)
        torch.testing.assert_close(e_fast, e_eager, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t_fast.reshape(-1), t_eager.reshape(-1), rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(e_torch, e_eager, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t_torch.reshape(-1), t_eager.reshape(-1), rtol=2e-4, atol=1e-6)
    assert o1._hgb_fast is not None                                  # the default took the captured path
    p1, p2, p3 = _flat_params(m1), _flat_params(m2), _flat_params(m3)
    assert _displacement_rel(p1, p2, p0) <= DISPLACEMENT_RTOL
    assert _displacement_rel(p2, p3, p0) <= DISPLACEMENT_RTOL


def test_train_recaptures_when_a_captured_hyperparameter_changes():
    """weight_decay and betas are kernel arguments of the captured step: after one epoch, changing them through param_groups
    makes hb.train capture again, so the fast path keeps following the eager one."""
    loader = _loader("qm9_painn", [24, 17, 31], with_edges=True)
    m1 = hb.get_distributed_model(hb.create_model(**ARCH["qm9_painn"]))
    m2 = copy.deepcopy(m1)
    p0 = _flat_params(m1).clone()
    o1, o2 = hb.FlatAdam(m1, lr=1e-3), hb.FlatAdam(m2, lr=1e-3)
    hb.train([b.clone() for b in loader], m1, o1)
    first = o1._hgb_fast
    hb.train([b.clone() for b in loader], m2, o2, fast=False)
    for o in (o1, o2):
        o.param_groups[0]["weight_decay"] = 0.5
        o.param_groups[0]["betas"] = (0.5, 0.9)
    e1, _ = hb.train([b.clone() for b in loader], m1, o1)
    e2, _ = hb.train([b.clone() for b in loader], m2, o2, fast=False)
    assert o1._hgb_fast is not None and o1._hgb_fast is not first
    torch.testing.assert_close(e1, e2, rtol=2e-4, atol=1e-6)
    assert _displacement_rel(_flat_params(m1), _flat_params(m2), p0) <= DISPLACEMENT_RTOL


@pytest.mark.parametrize("name,hp", CASES, ids=IDS)
def test_unaligned_buffers_take_the_scalar_path(name, hp):
    """Every buffer a view one element into its allocation (not 16-byte aligned): the kernel's scalar loop does the whole update,
    and gives the bits of the float4 path on aligned copies of the same data, and the fp64 oracle's values."""
    count, grad_scale = 4097, 0.25
    gen = torch.Generator(device=DEV).manual_seed(9)
    p0 = torch.randn(count, device=DEV, generator=gen)
    grads = [(torch.rand(count, device=DEV, generator=gen) + 0.5) * torch.randn(count, device=DEV, generator=gen).sign()
             for _ in range(STEPS)]
    init = {k: v.float() for k, v in oopt.new_state(name, p0.double(), **hp).items()}

    def shifted(t):
        buf = torch.empty(t.numel() + 1, device=DEV)
        view = buf[1:]
        view.copy_(t)
        assert view.data_ptr() % 16 != 0
        return view

    runs = []
    for make in (lambda t: t.clone(), shifted):
        p, st, step_dev = make(p0), {k: make(v) for k, v in init.items()}, torch.zeros(1, device=DEV)
        for g in grads:
            _launch(name, hp, p, make(g), st, step_dev, grad_scale)
        runs.append((p, st))
    (pa, sa), (pu, su) = runs
    assert torch.equal(pa, pu)
    for k in sa:
        assert torch.equal(sa[k], su[k])
    po, so = oracle_run(name, kernel_hp(name, hp), p0, grads, grad_scale=grad_scale)
    _close(pu, po)
    for k in so:
        _close(su[k], so[k])


def test_flat_adamw_captured_step_is_the_kernel_call_it_always_made():
    """FlatAdamW on the shared base: its captured step gives the parameters and moments of the direct hgb_adamw_step call
    sequence it made before the base existed, bit for bit, with lr changes between replays."""
    gen = torch.Generator(device=DEV).manual_seed(5)
    m = _toy(3)
    opt = hb.FlatAdamW(m, lr=1e-3)
    p, mm, v = opt.flat_p.clone(), torch.zeros_like(opt.flat_p), torch.zeros_like(opt.flat_p)
    step, hyper = torch.zeros(1, device=DEV), torch.tensor([1e-3, 1.0], device=DEV)
    warm = hb.FlatAdamW(_toy(4))
    warm.step()
    opt.sync_hyper(1.0)
    graph = torch.cuda.CUDAGraph()
    with ops.capture_graph(graph):
        opt.step()
    for t, lr in enumerate((1e-3, 1e-3, 5e-4, 1e-4)):
        g = torch.randn(opt.flat_g.shape, device=DEV, generator=gen)
        opt.flat_g.copy_(g)
        opt.param_groups[0]["lr"] = lr
        opt.sync_hyper()
        graph.replay()
        hyper.fill_(lr)
        hyper[1] = 1.0
        ops.adamw_step(p, g, mm, v, step, 0.0, 0.9, 0.999, 1e-8, 1e-2, 1.0, hyper_dev=hyper)
    torch.cuda.synchronize()
    assert torch.equal(opt.flat_p, p) and torch.equal(opt.m, mm) and torch.equal(opt.v, v) and torch.equal(opt.step_dev, step)
    assert opt.state_tensors()[0] is opt.m and opt.state_tensors()[-1] is opt.step_dev
