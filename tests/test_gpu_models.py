"""GPU parity tests, model level: the engine (through ``create_model``, the reference's plugin entry point)
against (a) the golden vectors produced by the reference's own code and (b) the CPU oracle on the synthetic
workloads, including forces (first-order path) and the MLIP double backward (any-order path).

Tolerance: fp32 engine vs fp32 reference/oracle, rel-L2 <= 1e-5 on outputs/forces (SURVEY 8d), elementwise
rtol 1e-4 on parameter gradients."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import ops  # noqa: E402
from hydragnn_b200.synthetic import ARCH, make_samples  # noqa: E402
import oracle  # noqa: E402
from oracle.workloads import add_edges_cpu  # noqa: E402
from stack_support import GPS_KW, HEAD_KW, MODEL_KW, PNAEQ_KW, _zero_dropout  # noqa: E402

DEV = "cuda"


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def _engine(kw, state):
    m = hb.create_model(**kw)
    inner = m.model if hasattr(m, "model") and isinstance(m, hb.create.EnhancedModelWrapper) else m
    inner.load_state_dict(state, strict=True)
    return m


def _batch(inputs, requires_pos_grad=False):
    d = hb.Batch(**{k: v.clone().to(DEV) for k, v in inputs.items()})
    d._num_graphs = int(inputs["batch"].max()) + 1
    if requires_pos_grad:
        d.pos.requires_grad_(True)
    return d


def test_create_model_reproduces_reference_initialisation(golden_dir):
    # same construction order + torch.manual_seed(0) => identical initial weights as the reference stack
    g = torch.load(golden_dir + "/models.pt")
    for name, kw in MODEL_KW.items():
        m = hb.create_model(**kw)
        sd = m.state_dict()
        assert list(sd.keys()) == list(g[name]["state"].keys()), name
        for k, v in sd.items():
            assert torch.equal(v.cpu(), g[name]["state"][k]), (name, k)


def test_unknown_mpnn_type_raises():
    with pytest.raises(ValueError):
        hb.create_model(**dict(MODEL_KW["egnn_mlip"], mpnn_type="NOPE"))


@pytest.mark.parametrize("name", list(MODEL_KW))
def test_forward_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models.pt")[name]
    m = _engine(MODEL_KW[name], c["state"]).eval()
    with torch.no_grad():
        pred = m(_batch(c["inputs"]))
    for p, q in zip(pred, c["pred"]):
        assert p.shape == q.shape
        assert rel_l2(p.cpu(), q) < 1e-5


@pytest.mark.parametrize("name", ["painn_graph_mean", "painn_graph_max"])
def test_painn_loss_and_param_grads_match_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models.pt")[name]
    m = _engine(MODEL_KW[name], c["state"]).train()
    d = _batch(c["inputs"])
    loss, _ = m.loss(m(d), d.y, [torch.arange(d.y.shape[0], device=DEV)])
    torch.testing.assert_close(loss.cpu(), c["loss"], rtol=1e-5, atol=1e-6)
    loss.backward()
    for n, p in m.named_parameters():
        ref = c["grads"][n]
        if ref is None:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, n
        else:
            torch.testing.assert_close(p.grad.cpu(), ref, rtol=2e-4, atol=1e-6, msg=lambda s, n=n: n + ": " + s)


@pytest.mark.parametrize("train_mode", [True, False])
def test_egnn_mlip_matches_reference_golden(golden_dir, train_mode):
    """train(): any-order path + double backward; eval(): fused first-order path (forces only)."""
    c = torch.load(golden_dir + "/models.pt")["egnn_mlip"]
    kw = dict(MODEL_KW["egnn_mlip"], enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0,
              force_weight=1.0)
    m = _engine(kw, c["state"])
    m.train(train_mode)
    d = _batch(c["inputs"], requires_pos_grad=True)
    pred = m(d)
    assert rel_l2(pred[0].cpu(), c["pred"][0]) < 1e-5
    tot, tasks = m.energy_force_loss(pred, d, create_graph=train_mode)
    torch.testing.assert_close(tot.detach().cpu(), c["loss"], rtol=1e-5, atol=1e-6)
    for a, b in zip(tasks, c["tasks"]):
        torch.testing.assert_close(a.detach().cpu(), b, rtol=1e-5, atol=1e-6)
    if train_mode:
        tot.backward()
        for n, p in m.model.named_parameters():
            ref = c["grads"][n]
            if ref is not None:
                torch.testing.assert_close(p.grad.cpu(), ref, rtol=5e-4, atol=1e-6, msg=lambda s, n=n: n + ": " + s)
    else:
        gcsr = d._hgb_gcsr
        e = ops.SegmentSum.apply(m(d)[0], ops.Csr(gcsr.idx, gcsr.rowptr, None, gcsr.n)).sum()
        f = -torch.autograd.grad(e, d.pos)[0]
        assert rel_l2(f.cpu(), c["forces"]) < 1e-5


def test_second_derivative_on_fused_path_raises(golden_dir):
    c = torch.load(golden_dir + "/models.pt")["egnn_mlip"]
    kw = dict(MODEL_KW["egnn_mlip"], enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0,
              force_weight=1.0)
    m = _engine(kw, c["state"]).eval()
    d = _batch(c["inputs"], requires_pos_grad=True)
    tot, _ = m.energy_force_loss(m(d), d, create_graph=True)
    with pytest.raises(RuntimeError):
        tot.backward()


# ---- synthetic workloads of the BASELINE shapes, engine vs oracle ------------------------------------------
def _pair(name, num_graphs):
    cpu = add_edges_cpu(make_samples(name, num_graphs), name)
    kw = ARCH[name]
    om = oracle.base.create_model(**kw)
    em = hb.create_model(**kw)
    inner = em.model if kw.get("enable_interatomic_potential") else em
    inner.load_state_dict((om.model if kw.get("enable_interatomic_potential") else om).state_dict())
    gpu = cpu.clone().to(DEV)
    gpu._num_graphs = num_graphs
    return cpu, gpu, om, em


def test_qm9_painn_training_step_matches_oracle():
    cpu, gpu, om, em = _pair("qm9_painn", 96)
    # edges from the engine's own radius-graph kernel must equal the oracle's, bit for bit
    eng = hb.get_radius_graph(7.0, 5)(gpu.clone())
    assert torch.equal(eng.edge_index.cpu(), cpu.edge_index)
    hi = [torch.arange(cpu.y.shape[0])]
    lo, _ = om.loss(om(cpu), cpu.y, hi)
    le, _ = em.loss(em(gpu), gpu.y, [hi[0].to(DEV)])
    torch.testing.assert_close(le.cpu(), lo.detach(), rtol=1e-5, atol=1e-6)
    lo.backward()
    le.backward()
    for (n, p), q in zip(em.named_parameters(), om.parameters()):
        torch.testing.assert_close(p.grad.cpu(), q.grad, rtol=5e-4, atol=1e-6, msg=lambda s, n=n: n + ": " + s)


@pytest.mark.parametrize("name,g", [("md17_egnn", 24), ("lj_egnn", 6)])
def test_mlip_training_step_matches_oracle(name, g):
    cpu, gpu, om, em = _pair(name, g)
    if name == "lj_egnn":   # periodic: the engine's batched PBC neighbour list equals the oracle's per-sample one
        eng = hb.get_radius_graph_pbc(5.0, 5)(gpu.clone())
        assert torch.equal(eng.edge_index.cpu(), cpu.edge_index)
        torch.testing.assert_close(eng.edge_shifts.cpu(), cpu.edge_shifts, rtol=0, atol=0)
    cpu.pos.requires_grad_(True)
    gpu.pos.requires_grad_(True)
    om.train()
    em.train()
    lo, to = om.energy_force_loss(om(cpu), cpu)
    le, te = em.energy_force_loss(em(gpu), gpu)
    torch.testing.assert_close(le.detach().cpu(), lo.detach(), rtol=1e-5, atol=1e-6)
    for a, b in zip(te, to):
        torch.testing.assert_close(a.detach().cpu(), b.detach(), rtol=1e-5, atol=1e-6)
    lo.backward()
    le.backward()
    for (n, p), q in zip(em.model.named_parameters(), om.model.parameters()):
        torch.testing.assert_close(p.grad.cpu(), q.grad, rtol=1e-3, atol=1e-6, msg=lambda s, n=n: n + ": " + s)


def test_force_equivariance_and_translation_invariance():
    """The reference's property test (tests/test_forces_equivariant.py:476: error < 1e-4): F(R x) = R F(x)."""
    for name in ("md17_egnn", "qm9_painn"):
        kw = dict(ARCH[name])
        if name == "qm9_painn":
            kw.update(output_type=["node"], output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [60, 20], "type": "mlp"}},
                      enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
        m = hb.create_model(**kw).eval()
        if name == "qm9_painn":
            # Reference quirk: update_U / update_V / vec_embed_out are nn.Linear WITH bias applied to every
            # Cartesian component of v (hydragnn/models/PAINNStack.py:281-282,98), which is not rotation-
            # equivariant unless the bias is zero.  The engine reproduces that arithmetic faithfully
            # (parity tests above); the property itself is checked with those biases zeroed.
            with torch.no_grad():
                for conv in m.model.graph_convs:
                    conv.module_1.update_U.bias.zero_()
                    conv.module_1.update_V.bias.zero_()
                    if hasattr(conv, "module_3"):
                        conv.module_3.bias.zero_()
        b = make_samples(name, 8).to(DEV)
        b._num_graphs = 8
        b = hb.get_radius_graph(7.0, 100000)(b)          # symmetric graph: rotation cannot change the edge set

        def forces(pos):
            d = b.clone()
            d._num_graphs = 8
            d.pos = pos.clone().requires_grad_(True)
            gc = None
            pred = m(d)
            gc = d._hgb_gcsr
            e = ops.SegmentSum.apply(pred[0], ops.Csr(gc.idx, gc.rowptr, None, gc.n))
            return -torch.autograd.grad(e.sum(), d.pos)[0], e.detach()

        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=torch.Generator().manual_seed(3)))
        q = q.to(DEV)
        f0, e0 = forces(b.pos)
        f1, e1 = forces(b.pos @ q.t() + torch.tensor([1.0, -2.0, 0.5], device=DEV))
        scale = float(f0.abs().max().clamp(min=1e-6))
        err = float((f1 - f0 @ q.t()).abs().max())
        # the reference's criterion is the ABSOLUTE max force error < 1e-4 (tests/test_forces_equivariant.py:476, "max_error < 1e-4");
        # the relative figure is kept as a second, looser bound (random-init forces are ~5e-3, fp32 rounding of O(1) activations ~1e-6)
        assert err < 1e-4 and err / scale < 5e-3, (name, err, err / scale)
        assert float((e1 - e0).abs().max()) / float(e0.abs().max().clamp(min=1e-6)) < 1e-4, name


def test_train_steps_reduce_loss_and_graphed_step_equals_eager():
    name, g = "qm9_painn", 256
    b = make_samples(name, g).to(DEV)
    b._num_graphs = g
    b = hb.get_radius_graph(7.0, 5)(b)
    model = hb.get_distributed_model(hb.create_model(**ARCH[name]))
    model2 = copy.deepcopy(model)
    opt = hb.FlatAdamW(model, lr=1e-3)
    losses = [float(hb.train_step(model, opt, b)[0]) for _ in range(30)]
    assert losses[-1] < losses[0]
    # CUDA-graph replay of the same step sequence gives the same losses (3 warm-up steps are part of the sequence)
    opt2 = hb.FlatAdamW(model2, lr=1e-3)
    gs = hb.GraphedTrainStep(model2, opt2, b.clone(), warmup=3)
    glosses = [float(gs.run()) for _ in range(27)]
    assert abs(glosses[-1] - losses[-1]) <= 1e-4 * abs(losses[-1]) + 1e-6


def test_validate_and_train_loop_api():
    name, g = "lj_egnn", 8
    b = make_samples(name, g).to(DEV)
    b._num_graphs = g
    b = hb.get_radius_graph_pbc(5.0, 5)(b)
    model = hb.get_distributed_model(hb.create_model(**ARCH[name]))
    opt = hb.FlatAdamW(model, lr=5e-3)
    e0, t0 = hb.validate([b.clone()], model, compute_grad_energy=True)
    for _ in range(5):
        err, terr = hb.train([b.clone()], model, opt, compute_grad_energy=True)
    e1, _ = hb.validate([b.clone()], model, compute_grad_energy=True)
    assert terr.shape == (3,) and float(e1) < float(e0)


# ---- PNAEq (row a6) ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["pnaeq_graph_mean", "pnaeq_graph_add"])
def test_pnaeq_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_pnaeq.pt")[name]
    kw = dict(PNAEQ_KW, graph_pooling=name.split("_")[-1], pna_deg=c["deg"])
    m = _engine(kw, c["state"]).train()
    d = _batch(c["inputs"])
    pred = m(d)
    assert rel_l2(pred[0].detach().cpu(), c["pred"][0]) < 1e-5
    loss, _ = m.loss(pred, d.y, [torch.arange(d.y.shape[0], device=DEV)])
    torch.testing.assert_close(loss.detach().cpu(), c["loss"], rtol=1e-5, atol=1e-6)
    loss.backward()
    for n, p in m.named_parameters():
        ref = c["grads"][n]
        if ref is not None:
            torch.testing.assert_close(p.grad.cpu(), ref, rtol=5e-4, atol=1e-6, msg=lambda s, n=n: n + ": " + s)


def test_pnaeq_mlip_double_backward_matches_oracle():
    name, g = "md17_egnn", 12
    cpu = add_edges_cpu(make_samples(name, g), name)
    deg = torch.bincount(torch.bincount(cpu.edge_index[1], minlength=cpu.pos.shape[0])).tolist()
    kw = dict(ARCH[name], mpnn_type="PNAEq", pna_deg=deg, num_radial=6, radius=7.0, hidden_dim=16)
    om = oracle.base.create_model(**kw)
    em = hb.create_model(**kw)
    em.model.load_state_dict(om.model.state_dict())
    gpu = cpu.clone().to(DEV)
    gpu._num_graphs = g
    cpu.pos.requires_grad_(True)
    gpu.pos.requires_grad_(True)
    om.train()
    em.train()
    lo, to = om.energy_force_loss(om(cpu), cpu)
    le, te = em.energy_force_loss(em(gpu), gpu)
    torch.testing.assert_close(le.detach().cpu(), lo.detach(), rtol=1e-5, atol=1e-6)
    lo.backward()
    le.backward()
    for (n, p), q in zip(em.model.named_parameters(), om.model.parameters()):
        if q.grad is not None:
            torch.testing.assert_close(p.grad.cpu(), q.grad, rtol=2e-3, atol=1e-6, msg=lambda s, n=n: n + ": " + s)


# ---- GPS global attention (row a9) ---------------------------------------------------------------------------
@pytest.mark.parametrize("n,f,heads", [(1, 8, 2), (77, 16, 4), (300, 64, 8), (1000, 64, 2), (129, 32, 32)])
def test_mha_kernel_matches_torch(n, f, heads):
    from hydragnn_b200.gps import MhaFn, mha_any_order
    g = torch.Generator().manual_seed(n + f)
    qkv = torch.randn(n, 3 * f, generator=g)
    go = torch.randn(n, f, generator=g)
    qr = qkv.clone().requires_grad_(True)
    q, k, v = [t.reshape(n, heads, f // heads).transpose(0, 1) for t in qr.split(f, dim=1)]
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).transpose(0, 1).reshape(n, f)
    gr, = torch.autograd.grad(ref, qr, go)
    qe = qkv.to(DEV).requires_grad_(True)
    out = MhaFn.apply(qe, heads)
    ge, = torch.autograd.grad(out, qe, go.to(DEV))
    torch.testing.assert_close(out.detach().cpu(), ref.detach(), rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(ge.cpu(), gr, rtol=1e-3, atol=1e-5)
    torch.testing.assert_close(mha_any_order(qe, heads).detach().cpu(), ref.detach(), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("name", ["gps_egnn", "gps_painn"])
def test_gps_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_gps.pt")[name]
    m = _engine(GPS_KW[name], c["state"])
    m.eval()
    with torch.no_grad():
        pred = m(_batch(c["inputs"]))
    assert rel_l2(pred[0].cpu(), c["pred_eval"][0]) < 1e-5
    m.train()
    _zero_dropout(m)
    d = _batch(c["inputs"])
    pred = m(d)
    assert rel_l2(pred[0].detach().cpu(), c["pred_train"][0]) < 1e-4
    loss, _ = m.loss(pred, d.y, [torch.arange(d.y.shape[0], device=DEV)])
    torch.testing.assert_close(loss.detach().cpu(), c["loss"], rtol=1e-4, atol=1e-6)
    loss.backward()
    for n, p in m.named_parameters():
        ref = c["grads"][n]
        if ref is not None:
            torch.testing.assert_close(p.grad.cpu(), ref, rtol=5e-3, atol=2e-5, msg=lambda s, n=n: n + ": " + s)
    sd = m.state_dict()
    for k, v in c["state_after"].items():
        torch.testing.assert_close(sd[k].cpu(), v, rtol=1e-4, atol=1e-6)


def test_gps_any_order_path_equals_fused_path(golden_dir):
    c = torch.load(golden_dir + "/models_gps.pt")["gps_painn"]
    m = _engine(GPS_KW["gps_painn"], c["state"]).eval()
    with torch.no_grad():
        a = m(_batch(c["inputs"]))[0]
        m.force_higher_order = True
        b = m(_batch(c["inputs"]))[0]
    assert rel_l2(b.cpu(), a.cpu()) < 1e-5


@pytest.mark.parametrize("name", list(HEAD_KW))
def test_node_heads_mlp_per_node_and_conv_match_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_heads.pt")[name]
    m = _engine(HEAD_KW[name], c["state"])
    m.train()
    d = _batch(c["inputs"])
    pred = m(d)
    assert rel_l2(pred[0].cpu(), c["pred"][0]) < 1e-5
    loss, _ = m.loss(pred, d.y, [torch.arange(d.y.shape[0], device=DEV)])
    assert abs(float(loss) - float(c["loss"])) < 1e-5 * max(1.0, abs(float(c["loss"])))
    loss.backward()
    gmax = max(float(v.abs().max()) for v in c["grads"].values() if v is not None)
    for n, p in m.named_parameters():
        ref = c["grads"][n]
        if ref is None:
            continue
        # biases in front of a BatchNorm have an exactly-zero gradient: compare on the scale of the whole gradient
        assert torch.allclose(p.grad.cpu(), ref, rtol=1e-3, atol=1e-4 * gmax), (name, n)
