"""CPU checks of the flat optimizers' host side: ``select_optimizer`` against the reference's own selection (tests/golden/optimizers.pt)
with and without ZeRO, its refusals, construction (conditioned models, parameters as views, torch's defaults and group keys), the
checkpoint format before any step, and a torch -> flat -> torch checkpoint round trip with the CUDA step replaced by the fp64 oracle
(the kernels themselves are checked in tests/test_gpu_optimizers.py)."""
import inspect

import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import ops
from optim_support import CASES, FLAT, IDS, TORCH
from oracle import optim as oopt
from stack_support import MACE_KW, MODEL_KW

TYPES = ("SGD", "Adam", "Adadelta", "Adagrad", "Adamax", "AdamW", "RMSprop")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir + "/optimizers.pt")


def _model():
    return hb.create_model(**dict(MODEL_KW["painn_graph_mean"], use_gpu=False))


@pytest.mark.parametrize("zero", [False, True])
@pytest.mark.parametrize("name", TYPES)
def test_select_optimizer_builds_what_the_reference_builds(golden, name, zero):
    rec = golden["types"][name]
    cfg = {"type": name, "learning_rate": golden["lr"]}
    if zero:
        cfg["use_zero_redundancy"] = True
    opt = hb.select_optimizer(_model(), cfg)
    assert isinstance(opt, hb.FlatOptimizer) and isinstance(opt, torch.optim.Optimizer)
    assert type(opt).__name__ == "Flat" + rec["class"]
    assert len(opt.param_groups) == 1
    group = opt.state_dict()["param_groups"][0]
    for k, v in rec["group"].items():
        assert group[k] == v, (k, group[k], v)


def test_select_optimizer_refusals(golden):
    ref = golden["errors"]["unknown"]
    with pytest.raises(NameError) as e:
        hb.select_optimizer(_model(), {"type": "Lion", "learning_rate": 1e-3})
    assert ref["type"] == "NameError" and str(e.value) == ref["msg"]
    with pytest.raises(ValueError, match="FusedLamb"):
        hb.select_optimizer(_model(), {"type": "FusedLAMB", "learning_rate": 1e-3})
    with pytest.raises(ValueError, match="FusedLamb"):
        hb.select_optimizer(_model(), {"type": "FusedLAMB", "learning_rate": 1e-3, "use_zero_redundancy": True})


@pytest.mark.parametrize("name", list(FLAT))
def test_keyword_defaults_are_torchs(name):
    flat = inspect.signature(FLAT[name].__init__).parameters
    ref = inspect.signature(TORCH[name].__init__).parameters
    for k, p in flat.items():
        if k in ("self", "model"):
            continue
        assert ref[k].default == p.default, (k, p.default, ref[k].default)


@pytest.mark.parametrize("name", list(FLAT))
def test_construction_refuses_a_conditioned_model_before_its_first_forward(name):
    kw = dict(MACE_KW, use_gpu=False, use_graph_attr_conditioning=True, graph_attr_conditioning_mode="film")
    m = hb.create_model(mpnn_type="MACE", **kw)
    with pytest.raises(ValueError, match="Flat%s: .*run one forward" % name):
        FLAT[name](m)


@pytest.mark.parametrize("name,hp", CASES, ids=IDS)
def test_parameters_become_views_and_state_dict_has_torchs_layout(name, hp):
    m = _model()
    before = {k: v.clone() for k, v in m.state_dict().items()}
    opt = FLAT[name](m, **hp)
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k])
    params = list(m.parameters())
    assert opt.flat_p.numel() == sum(p.numel() for p in params)
    opt.flat_p[:params[0].numel()] = 7.0
    assert float(params[0].detach().min()) == 7.0                          # parameters are views of the flat buffer
    ref = TORCH[name](_model().parameters(), **hp).state_dict()
    sd = opt.state_dict()
    assert sd["param_groups"][0].keys() == ref["param_groups"][0].keys()
    assert {k: v for k, v in sd["param_groups"][0].items()} == ref["param_groups"][0]
    assert sd["state"].keys() == ref["state"].keys()              # empty, except Adagrad's state from construction on
    for i, st in ref["state"].items():
        assert st.keys() == sd["state"][i].keys()
        for k, v in st.items():
            assert torch.equal(sd["state"][i][k], v) and sd["state"][i][k].dtype == v.dtype
    assert opt.state_tensors()[-1] is opt.step_dev
    assert len(opt.state_tensors()) == len(oopt.state_keys(name, **hp)) + 1


def _oracle_kernels(monkeypatch):
    """CPU stand-ins for the CUDA steps: the fp64 oracle on the flat buffers, lr / grad_scale from hyper_dev, step_dev counted."""
    def make(name, keys, hp_names):
        def f(p, g, *args, grad_scale=1.0, hyper_dev=None):
            bufs, step_dev, rest = args[:len(keys)], args[len(keys)], args[len(keys) + 1:]
            hp = dict(zip(hp_names, rest))
            if "beta1" in hp:
                hp["betas"] = (hp.pop("beta1"), hp.pop("beta2"))
            if hyper_dev is not None:
                hp["lr"], grad_scale = float(hyper_dev[0]), float(hyper_dev[1])
            st = {k: b.double() for k, b in zip(keys, bufs) if b is not None}
            pd = p.double()
            oopt.step(name, pd, g.double() * grad_scale, st, float(step_dev) + 1, **hp)
            p.copy_(pd)
            for k, b in zip(keys, bufs):
                if b is not None:
                    b.copy_(st[k])
            step_dev += 1
        return f
    monkeypatch.setattr(ops, "sgd_step", make("SGD", ["momentum_buffer"], ["lr", "momentum", "dampening", "nesterov", "weight_decay"]))
    monkeypatch.setattr(ops, "adam_step", make("Adam", ["exp_avg", "exp_avg_sq", "max_exp_avg_sq"],
                                               ["lr", "beta1", "beta2", "eps", "weight_decay", "amsgrad"]))
    monkeypatch.setattr(ops, "adamw_step", make("AdamW", ["exp_avg", "exp_avg_sq"], ["lr", "beta1", "beta2", "eps", "weight_decay"]))
    monkeypatch.setattr(ops, "adamax_step", make("Adamax", ["exp_avg", "exp_inf"], ["lr", "beta1", "beta2", "eps", "weight_decay"]))
    monkeypatch.setattr(ops, "adagrad_step", make("Adagrad", ["sum"], ["lr", "lr_decay", "weight_decay", "eps"]))
    monkeypatch.setattr(ops, "adadelta_step", make("Adadelta", ["square_avg", "acc_delta"], ["lr", "rho", "eps", "weight_decay"]))
    monkeypatch.setattr(ops, "rmsprop_step", make("RMSprop", ["square_avg", "momentum_buffer", "grad_avg"],
                                                  ["lr", "alpha", "eps", "weight_decay", "momentum", "centered"]))


@pytest.mark.parametrize("name,hp", CASES, ids=IDS)
def test_checkpoints_move_between_torch_and_flat_with_the_world_fold(monkeypatch, name, hp):
    """torch steps 3 times; its checkpoint goes into the flat optimizer, which steps 3 more times with a doubled gradient and
    grad_scale 0.5 (the 1/world fold of a 2-rank all-reduce); that checkpoint goes back into torch for 2 more steps.  Every leg
    equals torch stepping throughout."""
    _oracle_kernels(monkeypatch)
    gen = torch.Generator().manual_seed(11)
    grads = [[torch.randn(p.shape, generator=gen) for p in _model().parameters()] for _ in range(8)]
    ref_m = _model()
    ref = TORCH[name](ref_m.parameters(), **hp)

    def torch_steps(model, opt, steps):
        for s in steps:
            for p, g in zip(model.parameters(), grads[s]):
                p.grad = g.clone()
            opt.step()

    torch_steps(ref_m, ref, range(8))
    a = _model()
    oa = TORCH[name](a.parameters(), **hp)
    torch_steps(a, oa, range(3))
    b = _model()
    b.load_state_dict(a.state_dict())
    ob = FLAT[name](b, lr=123.0)
    ob.load_state_dict(oa.state_dict())
    assert ob.lr == hp["lr"]
    for s in range(3, 6):
        for p, g in zip(b.parameters(), grads[s]):
            p.grad = 2.0 * g
        ob.gather_grads()
        ob.step(grad_scale=0.5)
    c = _model()
    c.load_state_dict(b.state_dict())
    oc = TORCH[name](c.parameters(), lr=123.0)
    oc.load_state_dict(ob.state_dict())
    torch_steps(c, oc, range(6, 8))
    for p, q in zip(c.parameters(), ref_m.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("name", list(FLAT))
def test_reduce_lr_on_plateau_drives_the_lr_the_kernel_reads(monkeypatch, name):
    """ReduceLROnPlateau (train_validate_test.py:452-476 steps it) accepts a flat optimizer, and the lr it lowers reaches the
    device vector {lr, grad_scale} the kernel reads."""
    _oracle_kernels(monkeypatch)
    opt = FLAT[name](_model(), lr=1e-2)
    sched = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, mode="min", factor=0.5, patience=0)
    for p in opt.params:
        p.grad = torch.ones_like(p)
    opt.gather_grads()
    opt.step()
    sched.step(1.0)
    sched.step(2.0)
    assert opt.lr == 5e-3
    opt.sync_hyper()
    assert abs(float(opt.hyper_dev[0]) - 5e-3) < 1e-9


@pytest.mark.parametrize("flat,ref,kw,value", [("AdamW", "Adam", {}, "decoupled_weight_decay=False"),
                                               ("Adam", "AdamW", {}, "decoupled_weight_decay=True"),
                                               ("AdamW", "AdamW", dict(amsgrad=True), "amsgrad=True")])
def test_load_state_dict_refuses_a_checkpoint_of_another_algorithm(flat, ref, kw, value):
    """Adam's L2 decay, AdamW's decoupled decay and amsgrad are group values torch's checkpoints carry: one the flat step does not
    run is refused, not stepped as a different algorithm."""
    opt = FLAT[flat](_model())
    with pytest.raises(ValueError, match="Flat%s.load_state_dict: .* has %s," % (flat, value)):
        opt.load_state_dict(TORCH[ref](_model().parameters(), **kw).state_dict())


@pytest.mark.parametrize("name,key", [("SGD", "momentum"), ("RMSprop", "momentum"), ("RMSprop", "centered"), ("Adam", "amsgrad")])
def test_an_option_switched_on_through_param_groups_gets_its_state_buffer(monkeypatch, name, key):
    """momentum / centered / amsgrad set after construction: the next eager step allocates the buffer the update then reads, and
    ``captured_hyper()`` (what a captured step holds besides lr) reports the change, so ``train`` re-captures."""
    _oracle_kernels(monkeypatch)
    opt = FLAT[name](_model())
    before = opt.captured_hyper()
    opt.param_groups[0][key] = 0.9 if key == "momentum" else True
    assert opt.captured_hyper() != before
    for p in opt.params:
        p.grad = torch.ones_like(p)
    opt.gather_grads()
    opt.step()
    want = {"momentum": "momentum_buffer", "centered": "grad_avg", "amsgrad": "max_exp_avg_sq"}[key]
    assert want in opt.flat_state and len(opt.state_tensors()) == len(opt.buffer_keys()) + 1
    assert float(opt.flat_state[want].abs().sum()) > 0


@pytest.mark.parametrize("name", list(FLAT))
def test_load_state_dict_drops_the_captured_step(name):
    """A loaded checkpoint may bring other hyperparameters than the captured step holds: the cached padded step is dropped."""
    opt = FLAT[name](_model())
    opt._hgb_fast = object()
    opt.load_state_dict(TORCH[name](_model().parameters()).state_dict())
    assert opt._hgb_fast is None
