"""GPU tests of MACE graph-attribute conditioning: the graph-addend tensor-core Linear (hgb_tc_linear_graph_add) and the FiLM
kernels (hgb_film_fwd / hgb_film_bwd) one by one against fp64, the engine against the fp64 restatement
(oracle/mace.py) on first-order and MLIP double-backward passes, and hb.train's padded step carrying graph_attr."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import ops  # noqa: E402
from hydragnn_b200.synthetic import ARCH  # noqa: E402
from oracle.mace import MACEOracle  # noqa: E402
from oracle.mlip import MLIPWrapper  # noqa: E402
from oracle.workloads import add_edges_cpu  # noqa: E402
from stack_support import MACE_KW, _gpu_batch, _grad_rel, _loader, mace_batch, random_rotation  # noqa: E402
from hydragnn_b200.synthetic import make_samples  # noqa: E402

DEV = "cuda"


def rel_l2(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp(min=1e-30))


# graph sizes: single-atom graphs, an empty graph, a graph longer than one FiLM chunk (64 rows) and than one 64-row tile, and a
# total row count that is not a multiple of the tile
LAYOUTS = {"singles": [1] * 150, "mixed": [1, 0, 3, 200, 1, 17, 64, 65, 2], "long": [517, 1, 130]}


def _gcsr(sizes):
    batch = torch.cat([torch.full((k,), i, dtype=torch.int64) for i, k in enumerate(sizes)]).to(DEV)
    return batch, ops.graph_ptr_from_batch(batch, len(sizes))


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("g", [1, 3, 17])
@pytest.mark.parametrize("h", [32, 64, 128])
def test_graph_add_linear_matches_fp64(h, g, layout, exact):
    sizes = LAYOUTS[layout]
    gen = torch.Generator().manual_seed(h + 7 * g + len(sizes))
    batch, gcsr = _gcsr(sizes)
    n, ng = batch.numel(), len(sizes)
    x = torch.randn(n, h, generator=gen, dtype=torch.float64)
    w = torch.randn(h, h + g, generator=gen, dtype=torch.float64) / h ** 0.5
    b = torch.randn(h, generator=gen, dtype=torch.float64)
    ga = torch.randn(ng, g, generator=gen, dtype=torch.float64)
    ref = torch.cat([x, ga[batch.cpu()]], 1) @ w.T + b
    c = (ga @ w[:, h:].T + b).float().to(DEV)
    xd, wd = x.float().to(DEV).requires_grad_(True), w.float().to(DEV).requires_grad_(True)
    cd = c.clone().requires_grad_(True)
    with ops.tensor_cores(not exact):
        assert ops.graph_add_tc_ok(xd, wd[:, :h], cd)
        y = ops.GraphAddLinearFn.apply(xd, wd[:, :h], cd, gcsr)
        tol = 1e-5 if exact else 2e-2
        assert rel_l2(y, ref) < tol, rel_l2(y, ref)
        dy = torch.randn(n, h, generator=gen, dtype=torch.float64)
        y.backward(dy.float().to(DEV))
    assert rel_l2(xd.grad, dy @ w[:, :h]) < tol
    assert rel_l2(wd.grad[:, :h], dy.T @ x) < (1e-3 if exact else 2e-2)
    gc = torch.zeros(ng, h, dtype=torch.float64).index_add_(0, batch.cpu(), dy)
    assert rel_l2(cd.grad, gc) < 1e-5


def _film_ref(h, st, batch):
    c = h.shape[1]
    return h * (1 + torch.tanh(st[:, :c]))[batch] + st[:, c:][batch]


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("g", [1, 3, 17])
@pytest.mark.parametrize("h", [32, 64, 128])
def test_film_forward_backward_match_fp64_and_repeat_bitwise(h, g, layout):
    """g sets the conditioner's input width upstream; here it seeds the per-graph terms that the conditioner would produce."""
    sizes = LAYOUTS[layout]
    gen = torch.Generator().manual_seed(3 * h + g + len(sizes))
    batch, gcsr = _gcsr(sizes)
    n, ng = batch.numel(), len(sizes)
    x = torch.randn(n, h, generator=gen, dtype=torch.float64, requires_grad=True)
    st = (torch.randn(ng, g, generator=gen, dtype=torch.float64) @ torch.randn(g, 2 * h, generator=gen, dtype=torch.float64)
          / g ** 0.5).requires_grad_(True)
    ref = _film_ref(x, st, batch.cpu())
    dy = torch.randn(n, h, generator=gen, dtype=torch.float64)
    gx, gst = torch.autograd.grad(ref, (x, st), dy)
    runs = []
    for _ in range(2):
        xd, std = x.detach().float().to(DEV).requires_grad_(True), st.detach().float().to(DEV).requires_grad_(True)
        y = ops.FilmFn.apply(xd, std, gcsr)
        y.backward(dy.float().to(DEV))
        runs.append((y.detach(), xd.grad, std.grad))
    y, gxd, gstd = runs[0]
    assert rel_l2(y, ref) < 1e-6 and rel_l2(gxd, gx) < 1e-6 and rel_l2(gstd, gst) < 1e-5, (rel_l2(y, ref), rel_l2(gstd, gst))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    # the data-only pass (MLIP force pass) leaves out the per-graph sums
    xd, std = x.detach().float().to(DEV).requires_grad_(True), st.detach().float().to(DEV).requires_grad_(True)
    with ops.only_data_grads():
        gxo, gso = torch.autograd.grad(ops.FilmFn.apply(xd, std, gcsr), (xd, std), dy.float().to(DEV), allow_unused=True)
    assert torch.equal(gxo, gxd) and gso is None


# ---- engine against the fp64 restatement ---------------------------------------------------------------------------------
def _with_ga(d, gen, g=3, flat=False):
    ga = torch.randn(d.num_graphs, g, generator=gen, dtype=torch.float64)
    d.graph_attr = ga.reshape(-1) if flat else ga
    return d


def _pair(kw, seed=0):
    """Oracle and engine with the same (non-trivial) parameters, the conditioning modules created by a first forward."""
    torch.manual_seed(seed)
    o = MACEOracle(**kw)
    if kw["graph_attr_conditioning_mode"] == "film":
        o._ensure_graph_conditioner(3, torch.device("cpu"))
    elif kw["graph_attr_conditioning_mode"] == "concat_node":
        o._ensure_graph_concat_projector(3, o.hidden_dim, torch.device("cpu"))
    with torch.no_grad():
        for p in o.parameters():
            p.copy_(torch.randn_like(p) * (p.std() if p.numel() > 1 else 1.0))
    e = hb.create_model(mpnn_type="MACE", **kw)
    if kw["graph_attr_conditioning_mode"] == "film":
        e._ensure_graph_conditioner(3, e.device)
    elif kw["graph_attr_conditioning_mode"] == "concat_node":
        e._ensure_graph_concat_projector(graph_attr_dim=3, channel_dim=e.hidden_dim, device=e.device)
    e.load_state_dict(o.state_dict(), strict=True)
    return o.double(), e


def _to_dev(d, pos_grad=False):
    g = hb.Batch(x=d.x.float().to(DEV), pos=d.pos.detach().float().to(DEV), edge_index=d.edge_index.to(DEV), batch=d.batch.to(DEV),
                 graph_attr=d.graph_attr.float().to(DEV))
    g._num_graphs = d.num_graphs
    if pos_grad:
        g.pos.requires_grad_(True)
    return g


@pytest.mark.parametrize("higher", [False, True])
@pytest.mark.parametrize("mode", ["film", "concat_node"])
@pytest.mark.parametrize("hidden", [8, 32, 128])
def test_engine_matches_oracle_with_conditioning(hidden, mode, higher):
    kw = dict(MACE_KW, hidden_dim=hidden, use_graph_attr_conditioning=True, graph_attr_conditioning_mode=mode)
    o, e = _pair(kw)
    o.eval()
    if higher:
        e.train()
        e.force_higher_order = True
    else:
        e.eval()
    gen = torch.Generator().manual_seed(11)
    for flat in (False, True):
        dd = _with_ga(mace_batch(gen, sizes=(7, 9, 5)), gen, flat=flat)
        dd.pos.requires_grad_(True)
        ref = o(dd)
        g = _to_dev(dd, pos_grad=True)
        out = e(g)
        for a, b in zip(out, ref):
            assert a.shape == b.shape and rel_l2(a, b) < 1e-5, rel_l2(a, b)
        lo = ref[0].sum() + ref[1].pow(2).sum()
        le = out[0].sum() + out[1].pow(2).sum()
        fo, = torch.autograd.grad(lo, dd.pos, retain_graph=True, create_graph=higher)
        fe, = torch.autograd.grad(le, g.pos, retain_graph=True, create_graph=higher)
        assert rel_l2(fe, fo) < 1e-5, rel_l2(fe, fo)
        if higher:      # MLIP: the parameter gradients of a force loss (double backward)
            lo, le = lo + fo.pow(2).sum(), le + fe.pow(2).sum()
        o.zero_grad()
        e.zero_grad()
        lo.backward()
        le.backward()
        po, pe = dict(o.named_parameters()), dict(e.named_parameters())
        cond = [k for k in po if k.startswith("graph_")]
        assert cond
        for k, p in po.items():
            if p.grad is None or float(p.grad.abs().max()) == 0:
                continue
            assert rel_l2(pe[k].grad, p.grad) < 1e-3, (k, rel_l2(pe[k].grad, p.grad))
        for k in cond:
            assert po[k].grad is not None and float(po[k].grad.abs().max()) > 0, k


@pytest.mark.parametrize("mode", ["film", "concat_node"])
def test_engine_tf32_mode_with_conditioning_within_tolerance(mode):
    o, e = _pair(dict(MACE_KW, hidden_dim=64, use_graph_attr_conditioning=True, graph_attr_conditioning_mode=mode))
    hb.set_precision(e, "bf16")
    gen = torch.Generator().manual_seed(4)
    dd = _with_ga(mace_batch(gen, sizes=(70, 90, 50), box=9.0), gen)
    ref = o(dd)
    out = e(_to_dev(dd))
    for a, b in zip(out, ref):
        assert rel_l2(a, b) < 2e-2, rel_l2(a, b)


@pytest.mark.parametrize("mode", ["film", "concat_node"])
def test_conditioned_energy_is_invariant_and_forces_equivariant(mode):
    _, e = _pair(dict(MACE_KW, hidden_dim=32, output_dim=[1], output_type=["graph"], task_weights=[1.0],
                      use_graph_attr_conditioning=True, graph_attr_conditioning_mode=mode), seed=3)
    gen = torch.Generator().manual_seed(5)
    dd = _with_ga(mace_batch(gen), gen)
    rot = random_rotation(gen)
    g1 = _to_dev(dd, pos_grad=True)
    e1 = e(g1)[0]
    f1, = torch.autograd.grad(e1.sum(), g1.pos)
    d2 = hb.Batch(x=dd.x, pos=dd.pos @ rot.T, edge_index=dd.edge_index, batch=dd.batch, graph_attr=dd.graph_attr)
    d2._num_graphs = dd.num_graphs
    g2 = _to_dev(d2, pos_grad=True)
    e2 = e(g2)[0]
    f2, = torch.autograd.grad(e2.sum(), g2.pos)
    assert rel_l2(e2, e1) < 1e-5
    assert rel_l2(f2, f1 @ rot.T.float().to(DEV)) < 1e-4


def test_fuse_pool_outputs_are_bit_identical_to_an_unconditioned_model():
    kw = dict(MACE_KW, hidden_dim=32)
    plain = hb.create_model(mpnn_type="MACE", **kw)
    fused = hb.create_model(mpnn_type="MACE", use_graph_attr_conditioning=True, graph_attr_conditioning_mode="fuse_pool", **kw)
    fused.load_state_dict(plain.state_dict(), strict=True)
    gen = torch.Generator().manual_seed(8)
    dd = _with_ga(mace_batch(gen, sizes=(7, 9, 5)), gen)
    for a, b in zip(fused(_to_dev(dd)), plain(_to_dev(dd))):
        assert torch.equal(a, b)
    assert not [k for k in fused.state_dict() if k.startswith(("graph_conditioner", "graph_concat_projector"))]
    d0 = _to_dev(dd)
    d0.graph_attr = None
    with pytest.raises(ValueError, match="graph_attr is missing"):
        fused(d0)


def _gfm_kw(hidden=None):
    kw = dict(ARCH["gfm_mace"])
    if hidden:
        kw["hidden_dim"] = hidden
    return kw


def _gfm_attrs(b, gen):
    b.graph_attr = torch.randn(b.num_graphs, 2, generator=gen)
    return b


def test_gfm_mace_shape_mlip_step_with_edge_lengths_matches_oracle():
    """The gfm_mlip.json shape: MLIP wrapper, add pooling, edge_dim 1 = edge lengths, concat_node conditioning; losses and the
    double-backward parameter gradients, the projector's included."""
    name, g = "gfm_mace", 2
    cpu = add_edges_cpu(make_samples(name, g), name)
    gpu = _gpu_batch(cpu, name, g)
    assert torch.equal(gpu.edge_index.cpu(), cpu.edge_index)
    vec = cpu.pos[cpu.edge_index[1]] - cpu.pos[cpu.edge_index[0]] + cpu.edge_shifts.to(cpu.pos.dtype)
    cpu.edge_attr = vec.norm(dim=1, keepdim=True)
    gpu.edge_attr = cpu.edge_attr.float().to(DEV)
    gen = torch.Generator().manual_seed(2)
    cpu.graph_attr = torch.randn(g, 2, generator=gen, dtype=torch.float64)
    gpu.graph_attr = cpu.graph_attr.float().to(DEV)
    kw = _gfm_kw()
    torch.manual_seed(0)
    inner = {k: v for k, v in kw.items() if k not in ("mpnn_type", "enable_interatomic_potential", "energy_weight",
                                                       "energy_peratom_weight", "force_weight")}
    om = MLIPWrapper(MACEOracle(**inner), 0.0, 1.0, 10.0)
    em = hb.create_model(**kw)
    torch.manual_seed(7)
    om.model._ensure_graph_concat_projector(2, 128, torch.device("cpu"))
    em.model._ensure_graph_concat_projector(graph_attr_dim=2, channel_dim=128, device=em.model.device)
    em.model.load_state_dict(om.model.state_dict(), strict=True)
    om.train()
    em.train()
    cpu.pos.requires_grad_(True)
    gpu.pos.requires_grad_(True)
    lo, to = om.energy_force_loss(om(cpu), cpu)
    le, te = em.energy_force_loss(em(gpu), gpu)
    for a, b in zip(te, to):
        torch.testing.assert_close(a.detach().cpu().double(), b.detach().double(), rtol=1e-4, atol=1e-6)
    lo.backward()
    le.backward()
    assert _grad_rel(em.model, om.model) < 1e-3
    assert float(em.model.graph_concat_projector.weight.grad.abs().max()) > 0


# ---- hb.train's padded step carries graph_attr -----------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["film", "concat_node"])
def test_train_fast_path_equals_eager_conditioned_mace_mlip(mode):
    """A fresh conditioned model: one forward creates the modules, then FlatAdamW; the padded CUDA-graph step (zero graph_attr rows
    for its filler graphs, a new batch copied into the captured buffers every step) follows the eager path over two epochs."""
    loader = _loader("gfm_mace", [2, 1, 3, 2], with_edges=True)
    gen = torch.Generator().manual_seed(3)
    for i, bt in enumerate(loader):
        bt.y = None
        ga = torch.randn(bt.num_graphs, 2, generator=gen)
        bt.graph_attr = ga.reshape(-1) if i % 2 else ga          # both forms through collation and padding
    kw = dict(_gfm_kw(hidden=32), edge_dim=0, num_conv_layers=2, graph_attr_conditioning_mode=mode)
    m = hb.create_model(**kw)
    with pytest.raises(ValueError, match="run one forward"):
        hb.FlatAdamW(m)
    with torch.no_grad():
        d = loader[0].clone().to(DEV)
        d._num_graphs = loader[0].num_graphs
        m(d)
    m1 = hb.get_distributed_model(m)
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    for epoch in range(2):
        e_fast, t_fast = hb.train([b.clone() for b in loader], m1, o1, compute_grad_energy=True, fast=True)
        e_eager, t_eager = hb.train([b.clone() for b in loader], m2, o2, compute_grad_energy=True, fast=False)
        torch.testing.assert_close(e_fast, e_eager, rtol=2e-4, atol=1e-6)
        torch.testing.assert_close(t_fast.reshape(-1), t_eager.reshape(-1), rtol=2e-4, atol=1e-6)
