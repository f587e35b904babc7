"""Branch-weighted energies and forces of multi-branch interatomic potentials (``hb.branch_weighted_energy_forces``,
``hb.PaddedPredictStep``).

* The mix kernels (``hgb_branch_mix_fwd`` / ``_bwd``) against fp64 for B in {1, 2, 3, 16, 17}, graph and node forms, with no
  graphs and with a graph without atoms; the same bits on a second run; bad arguments refused before any launch.
* 3-branch EGNN and PaiNN potentials against the reference's own per-branch forward, ``_weighted_average`` and
  ``_fused_energy_forces`` (tests/golden/models_branch_mix.pt), PNAEq and MACE against oracle/branch_mix.py in fp64, for graph
  and node energy heads, at test_gpu_multibranch.py's tolerances.
* One-hot weights reproduce the model with ``dataset_name`` := b; one branch reproduces the MLIP prediction; one call with 16
  branches launches fewer than twice the kernels of a single-branch prediction; no parameter gradient or optimizer state
  changes.
* The captured step against the eager call over batches of changing size and weights, with one recapture.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops  # noqa: E402
from hydragnn_b200.stacks import Base  # noqa: E402
from hydragnn_b200.synthetic import ARCH  # noqa: E402
from oracle import base as obase  # noqa: E402
from oracle import branch_mix as obm  # noqa: E402
from stack_support import MACE_KW, _loader, mace_batch  # noqa: E402

DEV = "cuda"


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


def _p(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---- the mix kernels ------------------------------------------------------------------------------------------------------------
def _mix(e, w, gptr, g):
    r, b = e.shape
    out = torch.full((g,), float("nan"), device=DEV)
    eb = None if gptr is None else torch.full((g, b), float("nan"), device=DEV)
    _lib.call("hgb_branch_mix_fwd", _p(e), _p(gptr), _p(w), g, r, b, _p(eb), _p(out), _stream())
    seeds = torch.full((r, b), float("nan"), device=DEV)
    dout = torch.linspace(-1.0, 2.0, g, device=DEV)
    _lib.call("hgb_branch_mix_bwd", _p(dout), _p(gptr), _p(w), g, r, b, _p(seeds), _stream())
    return out, eb, seeds, dout


@pytest.mark.parametrize("form", ["graph", "node"])
@pytest.mark.parametrize("b", [1, 2, 3, 16, 17])
@pytest.mark.parametrize("counts", [[3, 0, 5, 1, 70, 2, 9, 4, 11], []])
def test_mix_kernels_match_fp64(form, b, counts):
    gen = torch.Generator().manual_seed(b * 7 + len(counts))
    g = len(counts)
    r = sum(counts) if form == "node" else g
    e = torch.randn(r, b, generator=gen, dtype=torch.float64)
    w = torch.softmax(torch.randn(g, b, generator=gen, dtype=torch.float64), dim=-1)
    graph_of = torch.repeat_interleave(torch.arange(g), torch.tensor(counts, dtype=torch.long)) if form == "node" else torch.arange(g)
    gptr = None
    if form == "node":
        gptr = torch.tensor([0] + torch.cumsum(torch.tensor(counts, dtype=torch.long), 0).tolist(), dtype=torch.int32, device=DEV)
    eb64 = torch.zeros(g, b, dtype=torch.float64).index_add_(0, graph_of, e)
    ef, wf = e.float().to(DEV), w.float().to(DEV)
    before = _lib.launch_count()
    out, eb, seeds, dout = _mix(ef, wf, gptr, g)
    assert _lib.launch_count() - before == (2 if g else 0)
    if g == 0:
        return
    torch.testing.assert_close(out.cpu().double(), (w * eb64).sum(1), rtol=1e-5, atol=1e-5)
    if eb is not None:
        torch.testing.assert_close(eb.cpu().double(), eb64, rtol=1e-5, atol=1e-5)
        assert float(eb[1].abs().max()) == 0.0 and float(out[1]) == 0.0            # the graph without atoms
    torch.testing.assert_close(seeds.cpu().double(), w[graph_of] * dout.cpu().double()[graph_of, None], rtol=1e-6, atol=1e-7)
    again = _mix(ef, wf, gptr, g)
    for a, c in zip((out, eb, seeds), again[:3]):
        assert a is None or torch.equal(a, c)                                        # the same bits on every run


def test_mix_kernels_empty_atoms_and_refusals():
    w = torch.rand(3, 4, device=DEV)
    gptr = torch.zeros(4, dtype=torch.int32, device=DEV)
    out, eb = torch.full((3,), float("nan"), device=DEV), torch.full((3, 4), float("nan"), device=DEV)
    before = _lib.launch_count()
    _lib.call("hgb_branch_mix_fwd", None, _p(gptr), _p(w), 3, 0, 4, _p(eb), _p(out), _stream())      # every graph empty
    _lib.call("hgb_branch_mix_bwd", _p(out), _p(gptr), _p(w), 3, 0, 4, None, _stream())
    assert _lib.launch_count() == before
    assert float(out.abs().max()) == 0.0 and float(eb.abs().max()) == 0.0
    e = torch.rand(5, 4, device=DEV)
    bad_fwd = [
        (_p(e), None, _p(w), 3, 5, 4, None, _p(out)),              # graph form: one row per graph
        (_p(e), _p(gptr), _p(w), 3, 5, 4, None, _p(out)),          # node form without eb
        (_p(e), None, None, 3, 3, 4, None, _p(out)),               # no weights
        (_p(e), None, _p(w), 3, 3, 4, None, None),                 # no output
        (None, None, _p(w), 3, 3, 4, None, _p(out)),               # no input
        (_p(e), None, _p(w), 3, 3, 0, None, _p(out)),              # no branch
        (_p(e), None, _p(w), -1, 3, 4, None, _p(out)),
        (_p(e), _p(gptr), _p(w), 3, -1, 4, _p(eb), _p(out)),
    ]
    bad_bwd = [
        (_p(out), None, _p(w), 3, 5, 4, _p(e)),
        (_p(out), _p(gptr), None, 3, 5, 4, _p(e)),
        (None, _p(gptr), _p(w), 3, 5, 4, _p(e)),
        (_p(out), _p(gptr), _p(w), 3, 5, 4, None),
        (_p(out), _p(gptr), _p(w), 3, 5, 0, _p(e)),
    ]
    before = _lib.launch_count()
    for args in bad_fwd:
        with pytest.raises(RuntimeError, match="bad arguments"):
            _lib.call("hgb_branch_mix_fwd", *args, _stream())
    for args in bad_bwd:
        with pytest.raises(RuntimeError, match="bad arguments"):
            _lib.call("hgb_branch_mix_bwd", *args, _stream())
    assert _lib.launch_count() == before


# ---- against the reference and the oracle ------------------------------------------------------------------------------------------
def _check(energy, forces, branch_energy, ref_energy, ref_forces, ref_branch):
    assert rel_l2(branch_energy, ref_branch) < 1e-5, rel_l2(branch_energy, ref_branch)
    assert rel_l2(energy, ref_energy) < 1e-5, rel_l2(energy, ref_energy)
    assert rel_l2(forces, ref_forces) < 1e-5, rel_l2(forces, ref_forces)


@pytest.mark.parametrize("name", ["egnn_graph", "egnn_node", "painn_graph", "painn_node"])
def test_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_branch_mix.pt")[name]
    e = hb.create_model(**c["cfg"], enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    e.model.load_state_dict(c["state"], strict=True)
    e.eval()
    d = hb.Batch(**{k: v.clone().to(DEV) for k, v in c["inputs"].items()})
    d._num_graphs = int(c["inputs"]["batch"].max()) + 1
    _lib.trace_begin()
    energy, forces, branch_energy = hb.branch_weighted_energy_forces(e, d, c["weights"].float().to(DEV))
    calls = {t[0] for t in _lib.trace_end()}
    assert {"hgb_grouped_linear", "hgb_branch_mix_fwd", "hgb_branch_mix_bwd"} <= calls
    _check(energy, forces, branch_energy, c["avg_energy"], c["avg_forces"], c["branch_energy"])
    _check(energy, forces, branch_energy, c["fused_energy"], c["fused_forces"], c["branch_energy"])


def _branches(arch, n=3):
    return [{"type": "branch-%d" % b, "architecture": dict(arch)} for b in range(n)]


GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 6]}
NODE = {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}
MLIP = dict(enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)


def _oracle_kw(stack, kind, d, n=3):
    kw = dict(output_dim=[1], output_type=[kind], task_weights=[1.0], loss_function_type="mse",
              output_heads={"graph": _branches(GRAPH, n), "node": _branches(NODE, n)},
              graph_pooling="add" if kind == "graph" else "mean", **MLIP)
    if stack == "MACE":
        return dict(MACE_KW, mpnn_type="MACE", **kw)
    deg = torch.bincount(torch.bincount(d.edge_index[1], minlength=d.pos.shape[0])).tolist()
    return dict(mpnn_type="PNAEq", input_dim=1, hidden_dim=12, activation_function="relu", num_conv_layers=3, num_radial=6,
                radius=5.0, pna_deg=deg, **kw)


def _engine_and_oracle(stack, kind, d, n=3):
    kw = _oracle_kw(stack, kind, d, n)
    o = obase.create_model(**kw)
    with torch.no_grad():
        for p in o.parameters():                               # make every path matter, as test_gpu_mace does
            p.copy_(torch.randn_like(p) * (p.std() if p.numel() > 1 else 1.0))
    e = hb.create_model(**kw)
    e.model.load_state_dict(o.model.state_dict(), strict=True)
    return e.eval(), o.double().eval()


def _gpu(d):
    g = hb.Batch(x=d.x.float().to(DEV), pos=d.pos.detach().float().to(DEV), edge_index=d.edge_index.to(DEV), batch=d.batch.to(DEV))
    g._num_graphs = d._num_graphs
    return g


@pytest.mark.parametrize("stack", ["PNAEq", "MACE"])
@pytest.mark.parametrize("kind", ["graph", "node"])
def test_matches_oracle(stack, kind):
    gen = torch.Generator().manual_seed(5)
    d = mace_batch(gen, sizes=(6, 8, 5, 7))
    e, o = _engine_and_oracle(stack, kind, d)
    w = torch.softmax(torch.randn(4, 3, generator=gen, dtype=torch.float64), dim=-1)
    g = _gpu(d)
    d.pos.requires_grad_(True)
    energies, forces = obm.per_branch(o, d, 3)
    e_avg, f_avg = obm.weighted_average(energies, forces, w, d.batch)
    e_fused, f_fused = obm.fused(o, d, w)
    energy, force, branch_energy = hb.branch_weighted_energy_forces(e, g, w.float().to(DEV))
    _check(energy, force, branch_energy, e_avg, f_avg, energies.T)
    _check(energy, force, branch_energy, e_fused, f_fused, energies.T)


# ---- special weights, launches, side effects ---------------------------------------------------------------------------------------
def _egnn_mlip(kind, n=3):
    kw = dict(ARCH["md17_egnn"], output_type=[kind], output_heads={"graph": _branches(GRAPH, n), "node": _branches(NODE, n)},
              graph_pooling="add" if kind == "graph" else "mean")
    return hb.create_model(**kw).eval()


def _one_branch(model, d, b):
    """``model(data)`` with ``dataset_name`` := b and its -dE/dpos, as the reference's per-branch loop computes them."""
    d.dataset_name = torch.full((d._num_graphs, 1), b, dtype=torch.long, device=DEV)
    pred = model(d)[0]
    if model.head_type[0] == "node":
        pred = ops.SegmentSum.apply(pred, Base.graph_index(d)[2])
    energy = pred.reshape(-1)
    with ops.only_data_grads():
        forces = -torch.autograd.grad(energy, d.pos, grad_outputs=torch.ones_like(energy))[0]
    del d.dataset_name
    return energy.detach(), forces


def _batch(sizes, seed=3):
    b = _loader("md17_egnn", [sizes], with_edges=True, seed0=seed)[0].to(DEV)
    b._num_graphs = sizes
    b.pos.requires_grad_(True)
    return b


@pytest.mark.parametrize("stack", ["EGNN", "MACE"])
@pytest.mark.parametrize("kind", ["graph", "node"])
def test_one_hot_weights_reproduce_each_branch(stack, kind):
    if stack == "EGNN":
        m, d = _egnn_mlip(kind), _batch(6)
    else:
        gen = torch.Generator().manual_seed(8)
        src = mace_batch(gen, sizes=(6, 8, 5, 7, 9, 4))
        m, d = _engine_and_oracle("MACE", kind, src)[0], _gpu(src)
        d.pos.requires_grad_(True)
    g = d._num_graphs
    for b in range(3):
        w = torch.zeros(g, 3, device=DEV)
        w[:, b] = 1.0
        energy, forces, branch_energy = hb.branch_weighted_energy_forces(m, d, w)
        ref_e, ref_f = _one_branch(m, d, b)
        torch.testing.assert_close(energy, ref_e, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(branch_energy[:, b], ref_e, rtol=1e-5, atol=1e-6)
        assert rel_l2(forces, ref_f) < 1e-5, rel_l2(forces, ref_f)


@pytest.mark.parametrize("kind", ["graph", "node"])
def test_one_branch_reproduces_the_mlip_prediction(kind):
    m, d = _egnn_mlip(kind, n=1), _batch(5)
    energy, forces, branch_energy = hb.branch_weighted_energy_forces(m, d, torch.ones(5, 1, device=DEV))
    pred = m(d)[0]
    ref_e = (ops.SegmentSum.apply(pred, Base.graph_index(d)[2]) if kind == "node" else pred).reshape(-1)
    ref_f = -torch.autograd.grad(ref_e, d.pos, grad_outputs=torch.ones_like(ref_e))[0]
    torch.testing.assert_close(energy, ref_e.detach(), rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(branch_energy[:, 0], ref_e.detach(), rtol=1e-6, atol=1e-6)
    assert rel_l2(forces, ref_f) < 1e-6


def test_one_encoder_pass_for_sixteen_branches():
    m, d = _egnn_mlip("graph", n=16), _batch(8)
    w = torch.softmax(torch.randn(8, 16, device=DEV), dim=-1)
    hb.branch_weighted_energy_forces(m, d, w)                   # warm: plans, modules
    _one_branch(m, d, 0)
    before = _lib.launch_count()
    hb.branch_weighted_energy_forces(m, d, w)
    mixed = _lib.launch_count() - before
    before = _lib.launch_count()
    _one_branch(m, d, 0)
    single = _lib.launch_count() - before
    assert 0 < mixed < 2 * single, (mixed, single)


def test_leaves_parameter_gradients_and_optimizer_state_alone():
    m, d = hb.get_distributed_model(_egnn_mlip("node")), _batch(6)
    opt = hb.FlatAdamW(m, lr=1e-3)
    m.train()
    t = d.clone()
    t.energy, t.forces = torch.randn(6, device=DEV), torch.randn(d.pos.shape[0], 3, device=DEV)
    t.dataset_name = torch.tensor([[0], [1], [2], [0], [1], [2]], device=DEV)
    hb.train_step(m, opt, t, compute_grad_energy=True)                     # gradients and optimizer state that are not zero
    m.eval()
    grads = {n: None if p.grad is None else p.grad.clone() for n, p in m.named_parameters()}
    state = [t.clone() for t in [opt.flat_p] + list(opt.state_tensors())]
    hb.branch_weighted_energy_forces(m, d, torch.softmax(torch.randn(6, 3, device=DEV), dim=-1))
    for n, p in m.named_parameters():
        assert (p.grad is None) == (grads[n] is None), n
        assert p.grad is None or torch.equal(p.grad, grads[n]), n
    for a, b in zip([opt.flat_p] + list(opt.state_tensors()), state):
        assert torch.equal(a, b)


# ---- the captured step -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["graph", "node"])
def test_captured_step_equals_eager(kind):
    m = _egnn_mlip(kind)
    loader = _loader("md17_egnn", [17, 9, 5, 31, 12], with_edges=True)       # the 31-graph batch outgrows the first capture
    step = hb.PaddedPredictStep(m, loader[0])
    gen = torch.Generator().manual_seed(1)
    for b in loader:
        g = int(b.batch.max()) + 1
        w = torch.softmax(torch.randn(g, 3, generator=gen), dim=-1)
        step.load(b, w)
        energy, forces, branch_energy = step.run()
        d = b.clone().to(DEV)
        d._num_graphs = g
        ref = hb.branch_weighted_energy_forces(m, d, w.to(DEV))
        assert energy.shape == (g,) and forces.shape == (b.pos.shape[0], 3) and branch_energy.shape == (g, 3)
        _check(energy, forces, branch_energy, ref[0], ref[1], ref[2])
    assert step.recaptures == 1
    step.check()
