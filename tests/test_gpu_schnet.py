"""SchNet on the H100: the fused CFConv kernels against the fp64 restatement, fused against composed, and the engine's SCFStack
against the reference's own stack (models_schnet.pt, written by tests/golden/make_schnet_golden.py)."""
import math

import pytest
import torch

from oracle import schnet as so
from conv_reference import cfconv as _fp64
from stack_support import _OD, _errors, _oracle, _oracle_step, golden_engine, rel_l2 as _rel

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _graph(gen, n=1200):
    """Isolated nodes, in-degrees 1, 2 and 1000, shuffled edge ids, edges longer than the cutoff (3.0)."""
    src, dst = [], []
    src += torch.randint(0, n, (1000,), generator=gen).tolist(); dst += [5] * 1000
    src += [7, 8, 9]; dst += [10, 11, 11]
    for i in range(20, n - 50):
        k = int(torch.randint(0, 5, (1,), generator=gen))
        src += torch.randint(0, n, (k,), generator=gen).tolist(); dst += [i] * k
    ei = torch.tensor([src, dst], dtype=torch.long)
    ei = ei[:, torch.randperm(ei.shape[1], generator=gen)]
    pos = torch.rand(n, 3, generator=gen, dtype=torch.float64) * 6.0
    return ei, pos


SHAPES = [(1, 2, 0), (8, 10, 1), (50, 50, 3), (64, 10, 16), (96, 10, 3), (126, 50, 0), (128, 50, 16), (128, 10, 3)]


def _setup(nf, g, d, seed=0):
    from hydragnn_b200 import ops
    gen = torch.Generator().manual_seed(seed)
    ei, pos = _graph(gen)
    n, e = pos.shape[0], ei.shape[1]
    mk = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64) * 0.5          # noqa: E731
    t = dict(xl=mk(n, nf), r=mk(e, d) if d else None, a1t=mk(g + d, nf), b1=mk(nf), w2=mk(nf, nf) / math.sqrt(nf), b2=mk(nf),
             g_out=mk(n, nf), g_we=mk(e, nf))
    offset = torch.linspace(0, 3.0, g, dtype=torch.float64)
    coeff = -0.5 / (3.0 / max(g - 1, 1)) ** 2
    plan = ops.EdgePlan(ei.to(DEV), n)
    return ei, pos, t, offset, coeff, plan


def _engine(ei, pos, t, offset, coeff, plan, cutoff=3.0):
    from hydragnn_b200 import ops
    f = {k: (v.float().to(DEV).requires_grad_(True) if v is not None and k not in ("g_out", "g_we") else v) for k, v in t.items()}
    p = pos.float().to(DEV).requires_grad_(True)
    out, w = ops.CfConvFn.apply(f["xl"], p, f["r"], f["a1t"], f["b1"], f["w2"], f["b2"], offset.float().to(DEV), coeff, cutoff,
                                plan, True)
    obj = (out * t["g_out"].float().to(DEV)).sum() + (w * t["g_we"].float().to(DEV)).sum()
    names = ["xl", "a1t", "b1", "w2", "b2"] + (["r"] if f["r"] is not None else [])
    grads = torch.autograd.grad(obj, [f[k] for k in names] + [p])
    return out, w, dict(zip(names + ["pos"], grads))


@pytest.mark.parametrize("nf,g,d", SHAPES)
def test_cfconv_kernels_against_fp64(nf, g, d):
    ei, pos, t, offset, coeff, plan = _setup(nf, g, d)
    out64, w64, g64 = _fp64(ei, pos, t, offset, coeff)
    out, w, gr = _engine(ei, pos, t, offset, coeff, plan)
    assert _rel(out.cpu(), out64) < 1e-5
    assert _rel(w.cpu(), w64) < 1e-5
    assert torch.all(out[torch.tensor([0, 1, 2, 3, 4]).to(DEV)] == 0)        # isolated nodes
    for k, ref in g64.items():
        assert _rel(gr[k].cpu(), ref) < 2e-5, (k, _rel(gr[k].cpu(), ref))


def test_cfconv_backward_is_bit_identical_across_runs():
    ei, pos, t, offset, coeff, plan = _setup(64, 10, 3, seed=3)
    a = _engine(ei, pos, t, offset, coeff, plan)
    b = _engine(ei, pos, t, offset, coeff, plan)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert all(torch.equal(a[2][k], b[2][k]) for k in a[2])


def test_cfconv_rejects_out_of_range_arguments():
    from hydragnn_b200 import _lib, ops
    assert ops.cfconv_supported(50, 126, 16) and ops.cfconv_supported(10, 8, 0)
    assert not ops.cfconv_supported(65, 64, 0) and not ops.cfconv_supported(10, 129, 0) and not ops.cfconv_supported(10, 64, 17)
    x = torch.zeros(4, 129, device=DEV)
    with pytest.raises(RuntimeError, match="cfconv_fwd: bad sizes"):
        _lib.call("hgb_cfconv_fwd", x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), None, None, 0, x.data_ptr(), -1.0, 3.0,
                  x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), 4, 0, 10, 129, x.data_ptr(), None, 0)


def _batch(case):
    from hydragnn_b200.data import Data
    d = Data(**{k: v.to(DEV) for k, v in case["inputs"].items()})
    return d


CASES = ["inlayer_graph", "inlayer_truncated", "equivariant_conv_head", "edge_len", "edge3", "gps", "gps_edge2", "add_pool"]


@pytest.mark.parametrize("higher", [False, True])
@pytest.mark.parametrize("name", CASES)
def test_engine_matches_the_reference_stack(golden_dir, name, higher):
    case = torch.load(golden_dir + "/models_schnet.pt")[name]
    m = golden_engine("SchNet", case)
    m.force_higher_order = higher
    m.eval()
    with torch.no_grad():
        pred = m(_batch(case))
    for p, ref in zip(pred, case["pred_eval"]):
        assert _rel(p.cpu(), ref) < 1e-5, name
    m.train()
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if hasattr(mod, "dropout") and isinstance(mod.dropout, float):
            mod.dropout = 0.0
    b = _batch(case)
    pred = m(b)
    value = case["value"].to(DEV)
    loss, _ = m.loss(pred, value, [torch.arange(value.numel(), device=DEV)])
    assert abs(float(loss) - float(case["loss"])) < 1e-5 * max(1.0, abs(float(case["loss"])))
    grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
    for (n, _), gr in zip(m.named_parameters(), grads):
        ref = case["grads"][n]
        if ref is None or float(ref.norm()) == 0:
            assert gr is None or float(gr.abs().max()) < 1e-6, n
            continue
        # a bias followed by BatchNorm has a zero true gradient: both sides hold rounding noise there
        err = float((gr.cpu().double() - ref.double()).norm())
        assert err <= 1e-4 * float(ref.double().norm()) + 1e-5, (name, n, err)


def test_nonzero_edge_shifts_do_not_change_the_result(golden_dir):
    case = torch.load(golden_dir + "/models_schnet.pt")["edge3"]
    m = golden_engine("SchNet", case).eval()
    b1, b2 = _batch(case), _batch(case)
    b2.edge_shifts = torch.zeros_like(b2.edge_shifts)
    with torch.no_grad():
        assert torch.equal(m(b1)[0], m(b2)[0])


def test_equivariant_layers_rebuild_the_graph_on_the_moved_positions(golden_dir):
    from hydragnn_b200 import ops, radius
    case = torch.load(golden_dir + "/models_schnet.pt")["equivariant_conv_head"]
    m = golden_engine("SchNet", case).eval()
    b = _batch(case)
    seen = []
    orig = ops.EdgePlan.__init__

    def spy(self, ei, *a, **k):
        seen.append(ei.clone())
        orig(self, ei, *a, **k)

    ops.EdgePlan.__init__ = spy
    try:
        with torch.no_grad():
            m(b)
    finally:
        ops.EdgePlan.__init__ = orig
    ref = case["graphs_eval"]                 # one per conv call: 3 encoder layers, 2 hidden and 1 output head conv
    # the last encoder layer does not move the atoms, so the first head conv reuses its graph: 5 builds for 6 calls
    assert len(ref) == 6 and len(seen) == 5
    for a, r in zip(seen, ref[:3] + ref[4:]):
        assert torch.equal(a.cpu(), r)


def _rot(seed):
    q, _ = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(seed), dtype=torch.float64))
    return q.float().to(DEV)


@pytest.mark.parametrize("head", ["conv", "mlp", "graph_add"])
def test_mlip_forces_rotate_with_the_input(golden_dir, head):
    import hydragnn_b200 as hb
    case = torch.load(golden_dir + "/models_schnet.pt")["equivariant_conv_head"]
    heads = {"conv": case["cfg"]["output_heads"],
             "mlp": {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [10, 6], "type": "mlp"}}]},
             "graph_add": {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5,
                                                                            "num_headlayers": 2, "dim_headlayers": [10, 7]}}]}}[head]
    m = hb.create_model(mpnn_type="SchNet", input_dim=1, hidden_dim=10, output_dim=[1], output_type=["graph" if head == "graph_add" else "node"],
                        output_heads=heads, num_conv_layers=3, num_filters=12, num_gaussians=8, radius=3.0, max_neighbours=20,
                        equivariance=True, graph_pooling="add" if head == "graph_add" else "mean", task_weights=[1.0],
                        enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    m.eval()
    b = _batch(case)

    def forces(pos):
        from hydragnn_b200.data import Data
        d = Data(x=b.x, pos=pos.clone().requires_grad_(True), batch=b.batch, energy=b.energy, forces=b.forces)
        e = m(d)[0]
        return -torch.autograd.grad(e.sum(), d.pos)[0]

    R = _rot(5)
    f0 = forces(b.pos)
    f1 = forces(b.pos @ R.t())
    assert _rel(f1, f0 @ R.t()) < 1e-4


def test_cfconv_backward_without_parameter_gradients():
    """Frozen filter parameters: the kernel skips the parameter sums, the data gradients are bit-identical."""
    from hydragnn_b200 import ops
    ei, pos, t, offset, coeff, plan = _setup(64, 10, 3, seed=4)
    _, _, full = _engine(ei, pos, t, offset, coeff, plan)
    f = {k: v.float().to(DEV) for k, v in t.items() if v is not None}
    xl, r = f["xl"].requires_grad_(True), f["r"].requires_grad_(True)
    p = pos.float().to(DEV).requires_grad_(True)
    out, w = ops.CfConvFn.apply(xl, p, r, f["a1t"], f["b1"], f["w2"], f["b2"], offset.float().to(DEV), coeff, 3.0, plan, True)
    obj = (out * f["g_out"]).sum() + (w * f["g_we"]).sum()
    gx, gr, gp = torch.autograd.grad(obj, [xl, r, p])
    assert torch.equal(gx, full["xl"]) and torch.equal(gr, full["r"]) and torch.equal(gp, full["pos"])


# ---- the fp64 oracle stack (oracle/schnet.py, itself checked against the reference's stack on the CPU) ------------------------
@pytest.mark.parametrize("nf,g", [(130, 10), (16, 65)])
def test_shapes_outside_the_kernel_run_composed_and_match_fp64(golden_dir, nf, g):
    import hydragnn_b200 as hb
    from hydragnn_b200 import _lib, ops
    assert not ops.cfconv_supported(g, nf, 0)
    case = torch.load(golden_dir + "/models_schnet.pt")["inlayer_graph"]
    kw = dict(mpnn_type="SchNet", input_dim=2, hidden_dim=12, output_dim=[1], output_type=["graph"],
              output_heads=case["cfg"]["output_heads"], num_conv_layers=2, num_filters=nf, num_gaussians=g, radius=3.0,
              max_neighbours=32, task_weights=[1.0])
    em = hb.create_model(**kw).train()
    state = {k: v.detach().cpu().clone() for k, v in em.state_dict().items()}
    b = _batch(case)
    _lib.trace_begin()
    pred = em(b)
    loss, _ = em.loss(pred, b.y.reshape(-1), [torch.arange(b.y.numel(), device=DEV)])
    loss.backward()
    calls = {c[0] for c in _lib.trace_end()}
    assert "hgb_cfconv_fwd" not in calls and "hgb_cfconv_bwd" not in calls
    om = _oracle(so.SCFStackOracle, kw, state).train()
    od = _OD(b)
    opred = om(od)
    oloss, _ = om.loss(opred, od.y.reshape(-1), [torch.arange(od.y.numel())])
    ograds = dict(zip([n for n, _ in om.named_parameters()], torch.autograd.grad(oloss, list(om.parameters()))))
    assert _rel(pred[0].detach().cpu(), opred[0].detach()) < 1e-5
    for n, p in em.named_parameters():
        ref = ograds[n]
        assert float((p.grad.cpu().double() - ref).norm()) <= 1e-4 * float(ref.norm()) + 1e-7, n


def test_mlip_forces_and_force_loss_gradients_match_fp64():
    """enable_interatomic_potential on the equivariant in-layer stack: forces (first order, fused path) and the parameter
    gradients of energy_force_loss (double backward, composed path) against the fp64 oracle with the reference's loss."""
    import hydragnn_b200 as hb
    from hydragnn_b200.synthetic import make_samples
    kw = dict(mpnn_type="SchNet", input_dim=1, hidden_dim=16, output_dim=[1], output_type=["node"], num_conv_layers=3,
              output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}}, num_filters=16,
              num_gaussians=10, radius=5.0, max_neighbours=20, equivariance=True, task_weights=[1.0])
    w = hb.create_model(**kw, enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    state = {k: v.detach().cpu().clone() for k, v in w.model.state_dict().items()}
    b = make_samples("ci_schnet", 32)
    w.eval()
    d = b.clone().to(DEV)
    d._num_graphs = 32
    d.pos.requires_grad_(True)
    f_eng = -torch.autograd.grad(w(d)[0].sum(), d.pos)[0]
    om = _oracle(so.SCFStackOracle, kw, state)
    od = _OD(b)
    od.pos.requires_grad_(True)
    f_ref = -torch.autograd.grad(om(od)[0].sum(), od.pos)[0]
    assert float(f_ref.norm()) > 0 and _rel(f_eng.cpu(), f_ref) < 1e-4
    w.train()
    d2 = b.clone().to(DEV)
    d2._num_graphs = 32
    d2.pos.requires_grad_(True)
    loss, _ = w.energy_force_loss(w(d2), d2)
    grads = torch.autograd.grad(loss, list(w.model.parameters()))
    om.train()
    od = _OD(b)
    od.pos.requires_grad_(True)
    e_node = om(od)[0]
    g = int(od.batch.max()) + 1
    e_graph = torch.zeros(g, dtype=torch.float64).index_add_(0, od.batch, e_node[:, 0])
    forces = -torch.autograd.grad(e_graph.sum(), od.pos, create_graph=True)[0]
    natoms = torch.bincount(od.batch, minlength=g).double()
    mse = torch.nn.functional.mse_loss
    ref_loss = mse(e_graph, od.energy) + mse(e_graph / natoms, od.energy / natoms) + mse(forces, od.forces)
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    rgrads = torch.autograd.grad(ref_loss, list(om.parameters()))
    eg = torch.cat([x.reshape(-1).double().cpu() for x in grads])
    rg = torch.cat([x.reshape(-1) for x in rgrads])
    assert _rel(eg, rg) < 1e-4


def _workload(name, graphs):
    from hydragnn_b200.synthetic import ARCH, add_rel_pe, make_samples
    from oracle.workloads import add_edges_cpu
    b = add_edges_cpu(make_samples(name, graphs), name)
    if ARCH[name].get("global_attn_engine"):
        add_rel_pe(b)
    return b, dict(ARCH[name])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name,graphs", [("qm9_schnet", 128), ("md17_schnet", 64), ("ci_schnet", 128)])
def test_training_step_at_workload_shape_matches_oracle(name, graphs, precision):
    """One training step against the fp64 oracle stack.  The oracle is also run at the engine's precision (fp32; for "bf16"
    fp32 with every Linear rounded to TF32) and measured against fp64: the engine must be within twice that and within the
    fixed bounds (fp32: outputs and loss rel-L2 1e-5, gradients 1e-4; TF32: 2e-2)."""
    import hydragnn_b200 as hb
    from hydragnn_b200 import _lib
    from oracle.tf32 import tf32_linears
    b, kw = _workload(name, graphs)
    em = hb.set_precision(hb.create_model(**kw), precision)
    for mod in em.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if hasattr(mod, "dropout") and isinstance(mod.dropout, float):
            mod.dropout = 0.0
    state = {k: v.detach().cpu().clone() for k, v in em.state_dict().items()}
    ref64 = _oracle_step(so.SCFStackOracle, kw, state, b, torch.float64)
    if precision == "fp32":
        ref32 = _errors(*_oracle_step(so.SCFStackOracle, kw, state, b, torch.float32), ref64)
    else:
        with tf32_linears():
            ref32 = _errors(*_oracle_step(so.SCFStackOracle, kw, state, b, torch.float32), ref64)
    em.train()
    d = b.clone().to(DEV)
    d._num_graphs = graphs
    _lib.trace_begin()
    pred = em(d)
    loss, _ = em.loss(pred, d.y.reshape(-1), [torch.arange(d.y.numel(), device=DEV)])
    loss.backward()
    calls = {t[0] for t in _lib.trace_end()}
    from hydragnn_b200.schnet import FUSED_MAX_FILTERS
    fused = kw["num_filters"] <= FUSED_MAX_FILTERS                   # ci_schnet (126 filters) runs the composed path
    assert ("hgb_cfconv_fwd" in calls and "hgb_cfconv_bwd" in calls) == fused, sorted(calls)
    eng = _errors(pred, loss.detach(), {n: p.grad for n, p in em.named_parameters()}, em.state_dict(), ref64)
    if precision == "fp32":
        bound = {"pred": max(1e-5, 2 * ref32["pred"]), "grad": max(1e-4, 2 * ref32["grad"]), "loss": max(1e-5, 2 * ref32["loss"])}
    else:
        bound = {k: max(2e-2, 2 * v) for k, v in ref32.items()}
    assert all(eng[k] <= bound[k] for k in eng), {"engine": eng, "oracle_same_precision": ref32, "bound": bound}


def test_hb_train_runs_schnet_eagerly_and_matches_the_eager_step():
    import copy
    import hydragnn_b200 as hb
    from hydragnn_b200 import padded
    b, kw = _workload("ci_schnet", 64)
    model = hb.get_distributed_model(hb.create_model(**kw))
    model2 = copy.deepcopy(model)
    assert not padded.supported(model)
    opt = hb.FlatAdamW(model, lr=1e-3)
    err, _ = hb.train([b.clone().to(DEV)], model, opt)
    opt2 = hb.FlatAdamW(model2, lr=1e-3)
    loss, _ = hb.train_step(model2, opt2, b.clone().to(DEV))
    assert abs(float(err) - float(loss)) <= 1e-6 * abs(float(loss))
    s1, s2 = model.module.state_dict(), model2.module.state_dict()
    for k in s1:
        torch.testing.assert_close(s1[k], s2[k], rtol=1e-6, atol=1e-8, msg=lambda m, k=k: k + ": " + m)
