"""GPU parity tests for the MACE path: engine (create_model(mpnn_type="MACE")) against the CPU oracle (oracle/mace.py,
run in float64) with the same weights on the same batch.  Tolerances: rel-L2 <= 1e-5 on outputs / forces (fp32 engine
vs fp64 oracle, SURVEY 8d); 1e-3 with the TF32 tensor-core Linears (precision="bf16")."""
import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from oracle import mace as omace  # noqa: E402
from oracle.mlip import MLIPWrapper  # noqa: E402
from stack_support import MACE_KW, mace_batch, random_rotation  # noqa: E402

DEV = "cuda"


def rel_l2(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp(min=1e-30))


def _pair(kw, seed=0):
    torch.manual_seed(seed)
    o = omace.MACEOracle(**kw)
    with torch.no_grad():
        for p in o.parameters():                      # make every path matter: fresh N(0,1)-scaled values
            p.copy_(torch.randn_like(p) * (p.std() if p.numel() > 1 else 1.0))
    e = hb.create_model(mpnn_type="MACE", **kw)
    e.load_state_dict(o.state_dict(), strict=True)
    return o.double(), e


def _to_dev(d, pos_grad=False):
    g = hb.Batch(x=d.x.float().to(DEV), pos=d.pos.float().to(DEV), edge_index=d.edge_index.to(DEV), batch=d.batch.to(DEV))
    g._num_graphs = d.num_graphs
    if pos_grad:
        g.pos.requires_grad_(True)
    return g


@pytest.mark.parametrize("variant", ["default", "ell3_corr3", "one_layer", "gaussian_add", "fused32", "fused64_ell3", "fused32_ell1", "fused128"])
def test_mace_forward_and_gradients_match_oracle(variant):
    kw = dict(MACE_KW)
    if variant == "ell3_corr3":
        kw.update(max_ell=3, node_max_ell=2, correlation=3, hidden_dim=4)
    elif variant == "one_layer":
        kw.update(num_conv_layers=1)
    elif variant == "gaussian_add":
        kw.update(radial_type="gaussian", graph_pooling="add", num_conv_layers=3, activation_function="sigmoid")
    elif variant == "fused32":            # channel counts % 32 == 0 take the fused tensor-product / contraction kernels
        kw.update(hidden_dim=32)
    elif variant == "fused64_ell3":
        kw.update(hidden_dim=64, max_ell=3, node_max_ell=2, num_conv_layers=3)
    elif variant == "fused128":            # two channel blocks per node in the tensor-product kernel
        kw.update(hidden_dim=128)
    elif variant == "fused32_ell1":
        kw.update(hidden_dim=32, max_ell=1, node_max_ell=1)
    o, e = _pair(kw)
    gen = torch.Generator().manual_seed(11)
    d = mace_batch(gen, sizes=(7, 9, 5))
    d.pos.requires_grad_(True)
    ref = o(d)
    g = _to_dev(d, pos_grad=True)
    out = e(g)
    for a, b in zip(out, ref):
        assert a.shape == b.shape and rel_l2(a, b) < 1e-5, (variant, rel_l2(a, b))
    # scalar objective -> forces and parameter gradients
    lo = ref[0].sum() + ref[1].pow(2).sum()
    le = out[0].sum() + out[1].pow(2).sum()
    fo, = torch.autograd.grad(lo, d.pos, retain_graph=True)
    fe, = torch.autograd.grad(le, g.pos, retain_graph=True)
    assert rel_l2(fe, fo) < 1e-5, rel_l2(fe, fo)
    lo.backward()
    le.backward()
    po, pe = dict(o.named_parameters()), dict(e.named_parameters())
    for k, p in po.items():
        if p.grad is None or float(p.grad.abs().max()) == 0:
            continue
        assert rel_l2(pe[k].grad, p.grad) < 2e-4, (variant, k, rel_l2(pe[k].grad, p.grad))


def test_mace_engine_rotation_invariance_and_force_equivariance():
    _, e = _pair(MACE_KW, seed=3)
    gen = torch.Generator().manual_seed(5)
    d = mace_batch(gen)
    rot = random_rotation(gen)
    g1 = _to_dev(d, pos_grad=True)
    o1 = e(g1)
    f1, = torch.autograd.grad(o1[0].sum() + o1[1].pow(2).sum(), g1.pos)
    d2 = hb.Batch(x=d.x, pos=d.pos @ rot.T + torch.tensor([0.3, -1.0, 2.0], dtype=torch.float64), edge_index=d.edge_index, batch=d.batch)
    d2._num_graphs = d.num_graphs
    g2 = _to_dev(d2, pos_grad=True)
    o2 = e(g2)
    f2, = torch.autograd.grad(o2[0].sum() + o2[1].pow(2).sum(), g2.pos)
    assert rel_l2(o2[0], o1[0]) < 1e-5 and rel_l2(o2[1], o1[1]) < 1e-4
    assert rel_l2(f2, f1 @ rot.float().to(DEV).T) < 1e-4                     # tests/test_forces_equivariant.py:476


def test_mace_mlip_double_backward_matches_oracle():
    kw = dict(MACE_KW, output_dim=[1], output_type=["node"], task_weights=[1.0],
              output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}},
              enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0,
              loss_function_type="mse")
    torch.manual_seed(0)
    o = omace.MACEOracle(**kw)
    e = hb.create_model(mpnn_type="MACE", **kw)
    e.model.load_state_dict(o.state_dict(), strict=True)
    ow = MLIPWrapper(o.double(), 1.0, 1.0, 1.0)
    gen = torch.Generator().manual_seed(2)
    d = mace_batch(gen, sizes=(6, 8))
    d.energy = torch.randn(2, generator=gen, dtype=torch.float64)
    d.forces = torch.randn(14, 3, generator=gen, dtype=torch.float64)
    d.pos.requires_grad_(True)
    lo, to = ow.energy_force_loss(ow(d), d)
    lo.backward()
    g = _to_dev(d, pos_grad=True)
    g.energy, g.forces = d.energy.float().to(DEV), d.forces.float().to(DEV)
    e.train()
    le, te = e.energy_force_loss(e(g), g)
    le.backward()
    assert abs(float(le) - float(lo)) < 1e-5 * max(1.0, abs(float(lo)))
    for a, b in zip(te, to):
        assert abs(float(a) - float(b)) < 1e-5 * max(1.0, abs(float(b)))
    po, pe = dict(o.named_parameters()), dict(e.model.named_parameters())
    for k, p in po.items():
        if p.grad is None or float(p.grad.abs().max()) < 1e-12:
            continue
        assert rel_l2(pe[k].grad, p.grad) < 5e-4, (k, rel_l2(pe[k].grad, p.grad))


def test_mace_bf16_mode_within_tolerance():
    o, e = _pair(dict(MACE_KW, hidden_dim=64, num_radial=8))
    hb.set_precision(e, "bf16")
    gen = torch.Generator().manual_seed(4)
    d = mace_batch(gen, sizes=tuple([9] * 40), box=5.0)
    ref = o(d)
    out = e(_to_dev(d))
    for a, b in zip(out, ref):
        assert rel_l2(a, b) < 2e-2


@pytest.mark.parametrize("name", ["mace_l2_nu2", "mace_l2_nu3", "mace_l3_nu2", "mace_one_layer"])
def test_mace_engine_matches_the_reference_own_code_golden(golden_dir, name):
    """tests/golden/models_mace.pt comes from the reference's own MACE files (e3nn stubbed by the oracle's restatement)."""
    c = torch.load(golden_dir + "/models_mace.pt")[name]
    kw = dict(MACE_KW, **c["cfg"])
    e = hb.create_model(mpnn_type="MACE", **kw)
    assert list(e.state_dict().keys()) == list(c["state"].keys())
    e.load_state_dict(c["state"], strict=True)
    e.eval()
    d = hb.Batch(**{k: v.clone().to(DEV) for k, v in c["inputs"].items()})
    d._num_graphs = 3
    d.pos.requires_grad_(True)
    pred = e(d)
    for p, q in zip(pred, c["pred"]):
        assert rel_l2(p, q) < 1e-5
    obj = pred[0].sum() + pred[1].pow(2).sum()
    f, = torch.autograd.grad(obj, d.pos, retain_graph=True)
    assert rel_l2(f, c["dobj_dpos"]) < 1e-4
    obj.backward()
    for n, p in e.named_parameters():
        ref = c["grads"][n]
        if ref is None or float(ref.abs().max()) == 0:
            continue
        assert rel_l2(p.grad, ref) < 5e-4, (name, n, rel_l2(p.grad, ref))
