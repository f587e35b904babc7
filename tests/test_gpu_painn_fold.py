"""GPU tests of the affine-v PaiNN message (PainnMessageFn given v0, w, b instead of v = Linear(1, 64)(v0)).
The reference is the composed path, ``linear_act`` then the message kernels on the stored v: every output and every gradient,
vec_embed_out's weight and bias gradients included, must keep its bits, so that training follows the same trajectory."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200 import _lib, ops  # noqa: E402
from hydragnn_b200.synthetic import ARCH, make_samples  # noqa: E402

DEV = "cuda"
F, R = 64, 5


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm())


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def make_case(n, graph, seed, edge_dim=None):
    """n atoms in graphs of ``graph`` atoms, every pair within a graph an edge, edge ids shuffled"""
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    gid = torch.arange(n) // graph
    start = gid * graph
    size = torch.minimum(torch.full((n,), graph), n - start)
    k = min(graph - 1, 12)                               # neighbours per atom: the next k atoms of its graph (cyclic)
    off = torch.arange(1, k + 1)
    src = torch.arange(n).repeat_interleave(k)
    dst = start.repeat_interleave(k) + (src - start.repeat_interleave(k) + off.repeat(n)) % size.repeat_interleave(k)
    ei = torch.stack([dst, src])
    ei = ei[:, ei[0] != ei[1]]
    ei = ei[:, torch.randperm(ei.shape[1], generator=g)].to(DEV)
    pos = (torch.randn(n, 3, generator=g) + 4.0 * gid[:, None]).to(DEV)
    plan = ops.EdgePlan(ei, n)
    _, ln, unit = ops.EdgeGeomFn.apply(pos, None, plan, 1e-9)
    epack = ops.PainnEdgeEmbedFn.apply(unit, ln, R, 7.0).detach()
    t = lambda *shape: torch.randn(*shape, generator=g).to(DEV)  # noqa: E731
    case = dict(phi=t(n, 3 * F), s=t(n, F), v0=t(n, 3, 1), w=t(F, 1), b=t(F), wf=t(3 * F, R) * 0.3, bf=t(3 * F),
                efilt=t(ei.shape[1], 3 * F) if edge_dim else None, gs=t(n, F), gv=t(n, 3, F), epack=epack, plan=plan)
    case["rec"] = ops.painn_edge_records(epack, plan, "row")
    return case


def run(c, fold):
    """outputs and gradients: s_out, v_out, gphi, gs, gv0, gw, gb, gwf, gbf, g_epack (+ g_efilt)"""
    leaves = {k: c[k].clone().requires_grad_(True) for k in ("phi", "s", "v0", "w", "b", "wf", "bf", "epack")}
    ef = c["efilt"].clone().requires_grad_(True) if c["efilt"] is not None else None
    L = leaves
    if fold:
        v = ops.AffineV(L["v0"], L["w"], L["b"])
        assert ops.painn_affine_v_ok(v, L["s"], c["rec"])
        s1, v1 = ops.PainnMessageFn.apply(L["phi"], L["s"], None, L["epack"], L["wf"], L["bf"], ef, c["plan"], c["rec"], *v)
        vin = None
    else:
        vin = ops.linear_act(L["v0"], L["w"], L["b"])
        s1, v1 = ops.PainnMessageFn.apply(L["phi"], L["s"], vin, L["epack"], L["wf"], L["bf"], ef, c["plan"], c["rec"])
    wrt = [L[k] for k in ("phi", "s", "v0", "w", "b", "wf", "bf", "epack")] + ([ef] if ef is not None else [])
    if vin is not None:
        wrt.append(vin)
    grads = torch.autograd.grad((s1 * c["gs"]).sum() + (v1 * c["gv"]).sum(), wrt)
    torch.cuda.synchronize()
    out = [s1.detach(), v1.detach()] + list(grads)
    if vin is None:
        return out, None
    return out[:-1], out[-1]           # the composed path also returns gv1, the gradient of the stored v


NAMES = ["s_out", "v_out", "gphi", "gs", "gv0", "gw", "gb", "gwf", "gbf", "g_epack", "g_efilt"]


@pytest.mark.parametrize("n,graph,edge_dim", [(256, 9, None), (257, 9, None), (4099, 9, None), (147456, 9, None),
                                              (4099, 200, None), (4099, 9, 3)])
def test_affine_v_message_same_bits_as_composed(n, graph, edge_dim):
    c = make_case(n, graph, seed=n + graph, edge_dim=edge_dim)
    fold, _ = run(c, True)
    ref, gv1 = run(c, False)
    again, _ = run(c, True)
    for name, x, r, y in zip(NAMES, fold, ref, again):
        assert same_bits(x, y), "%s differs between two runs" % name
        assert same_bits(x, r), "%s differs from the composed path: rel-L2 %.3g" % (name, rel(x, r))
    # vec_embed_out's gradients in fp64 from the stored gv1 of the composed path
    g64, x64 = gv1.double(), c["v0"].double()
    gw64 = (g64 * x64).sum(dim=(0, 1)).reshape(F, 1)
    gb64 = g64.sum(dim=(0, 1))
    assert rel(fold[5], gw64) <= 1e-5 and rel(fold[6], gb64) <= 1e-5, (rel(fold[5], gw64), rel(fold[6], gb64))


def _batch(name, graphs, **arch):
    kw = dict(ARCH[name], **arch)
    torch.manual_seed(0)
    m = hb.create_model(**kw).to(DEV)
    b = make_samples(name, graphs).to(DEV)
    b._num_graphs = graphs
    b = hb.get_radius_graph(7.0, 5)(b)
    return m, b


def _step(m, b, tc, force_higher=False):
    """loss, parameter gradients and the traced C-ABI calls of one forward / backward"""
    m.zero_grad(set_to_none=True)
    m.force_higher_order = force_higher
    hi = [torch.arange(b._num_graphs, device=DEV)]
    _lib.trace_begin()
    try:
        with ops.tensor_cores(tc):
            loss, _ = m.loss(m(b), b.y, hi)
            loss.backward()
        torch.cuda.synchronize()
    finally:
        calls = _lib.trace_end()
    return loss.detach(), [p.grad.detach().clone() for p in m.parameters()], calls


def _vec_embed_calls(calls, n):
    """(small-k forward calls on the [3N, 1] layer-0 v, small-k backward calls on it, message calls given v0)"""
    sk = [[a for name, a, _ in calls if name == entry and a["m"] == 3 * n and a["k"] == 1]
          for entry in ("hgb_linear_smallk_fwd", "hgb_linear_smallk_bwd")]
    av = [a for name, a, _ in calls if name in ("hgb_painn_message_fwd", "hgb_painn_message_bwd") and a["v_in"]]
    return sk[0], sk[1], av


@pytest.mark.parametrize("hidden,graphs,folded", [(64, 64, True), (32, 64, False), (64, 20, False)])
def test_painn_fold_dispatch(hidden, graphs, folded):
    """the C2 model forms layer 1's v inside the message kernels (only the small-k backward remains, on gv); hidden width 32
    and n < 256 keep the Linear(1, F) forward"""
    m, b = _batch("qm9_painn", graphs, hidden_dim=hidden)
    n = b.x.shape[0]
    _, _, calls = _step(m, b, False)
    fwd, bwd, av = _vec_embed_calls(calls, n)
    assert len(bwd) == 1
    if folded:
        assert not fwd and len(av) == 2
    else:
        assert len(fwd) == 1 and not av


def test_painn_fold_not_taken_on_higher_order_path():
    """the any-order path materialises v with its own closed primitives and agrees with the folded first-order step"""
    m, b = _batch("qm9_painn", 64)
    loss_h, grads_h, calls = _step(m, b, False, force_higher=True)
    assert not _vec_embed_calls(calls, b.x.shape[0])[2]
    loss_f, grads_f, _ = _step(m, b, False)
    assert abs(float(loss_h) - float(loss_f)) <= 1e-4 * abs(float(loss_f))
    assert rel(torch.cat([g.flatten() for g in grads_h]), torch.cat([g.flatten() for g in grads_f])) <= 1e-4


def test_painn_fold_trains_on_flat_parameters(monkeypatch):
    """FlatAdamW makes every parameter a view of one flat buffer (vec_embed_out's weight and bias are then only 4-byte
    aligned); twenty AdamW steps follow the composed path's trajectory bit for bit"""
    runs = []
    for fold in (True, False):
        if not fold:
            monkeypatch.setattr(ops, "painn_affine_v_ok", lambda *a: False)
        m, b = _batch("qm9_painn", 512)
        model = hb.get_distributed_model(m)
        opt = hb.FlatAdamW(model, lr=1e-3)
        losses = [hb.train_step(model, opt, b)[0].detach().clone() for _ in range(20)]
        torch.cuda.synchronize()
        runs.append((losses, [p.detach().clone() for p in m.parameters()]))
    for i, (a, c) in enumerate(zip(runs[0][0], runs[1][0])):
        assert same_bits(a, c), "step %d: loss %r vs %r" % (i, float(a), float(c))
    for (name, _), a, c in zip(m.named_parameters(), runs[0][1], runs[1][1]):
        assert same_bits(a, c), "%s differs after 20 steps: rel-L2 %.3g" % (name, rel(a, c))


@pytest.mark.parametrize("tc", [False, True])
def test_painn_model_fold_matches_composed(tc, monkeypatch):
    """a C2-shaped model: the loss and every parameter gradient keep the composed path's bits"""
    m, b = _batch("qm9_painn", 2048)
    loss_f, grads_f, calls = _step(m, b, tc)
    assert _vec_embed_calls(calls, b.x.shape[0])[2]
    monkeypatch.setattr(ops, "painn_affine_v_ok", lambda *a: False)
    loss_c, grads_c, calls = _step(m, b, tc)
    assert not _vec_embed_calls(calls, b.x.shape[0])[2]
    assert same_bits(loss_f, loss_c), (float(loss_f), float(loss_c))
    for (name, _), gf, gc in zip(m.named_parameters(), grads_f, grads_c):
        assert same_bits(gf, gc), "%s: rel-L2 %.3g" % (name, rel(gf, gc))
