"""CPU checks of the PNAPlus restatements (oracle/pnaplus.py) and of the engine's seeded construction.

models_pnaplus.pt pins the reference's own PNAPlusStack.py / Base.py with PyG's BesselBasisLayer / Envelope restated, so the
basis is pinned here by hand-computed values and derivatives (d/d dist and d/d freq), and the oracle stack is checked against
every golden case it restates (no GPS, no conv-type heads).
"""
import math

import pytest
import torch

from oracle.base import oracle_from_case
from oracle.pnaplus import BesselBasisLayer, Envelope
from stack_support import check_golden_case, check_grads, check_seeded_state, golden_data, grad_close

CASES = ["pnaplus_graph_noedge", "pnaplus_node_edge_len", "pnaplus_multihead_h5", "pnaplus_gps", "pnaplus_edge_dim0",
         "pnaplus_add_pool_edge3", "pnaplus_conv_head"]


def _env(x, e):
    """env(x) and env'(x) written out for exponent e: p = e + 1."""
    p = e + 1
    a, b, c = -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2
    if x >= 1.0:
        return 0.0, 0.0
    return (1 / x + a * x ** (p - 1) + b * x ** p + c * x ** (p + 1),
            -1 / x ** 2 + a * (p - 1) * x ** (p - 2) + b * p * x ** (p - 1) + c * (p + 1) * x ** p)


def test_envelope_hand_values():
    # exponent 5: p = 6, a = -28, b = 48, c = -21; at x = 1/2: 2 - 28/32 + 48/64 - 21/128 = 1.7109375
    env = Envelope(5)
    assert (env.p, env.a, env.b, env.c) == (6, -28.0, 48, -21.0)
    x = torch.tensor([0.5, 1.0, 1.5], dtype=torch.float64)
    torch.testing.assert_close(env(x), torch.tensor([1.7109375, 0.0, 0.0], dtype=torch.float64), rtol=0, atol=1e-15)
    # the envelope and its first two derivatives vanish at x = 1 from below
    y = torch.tensor([1.0 - 1e-6], dtype=torch.float64)
    assert abs(float(env(y))) < 1e-12


@pytest.mark.parametrize("expo", [1, 3, 5])
def test_bessel_basis_values_and_derivatives(expo):
    r, cutoff = 4, 2.5
    layer = BesselBasisLayer(r, cutoff, expo).double()
    # initialised in fp32 (before .double()): pi (1..R) rounded to fp32
    torch.testing.assert_close(layer.freq.detach(), (math.pi * torch.arange(1, r + 1, dtype=torch.float64)).float().double(), rtol=0, atol=0)
    fr = layer.freq.detach().tolist()
    dist = torch.tensor([0.3, 1.1, 2.4, 2.5, 3.7], dtype=torch.float64, requires_grad=True)
    rbf = layer(dist)
    for i, d in enumerate(dist.tolist()):
        x = d / cutoff
        e, de = _env(x, expo)
        for k in range(r):
            f = fr[k]
            assert abs(float(rbf[i, k].detach()) - e * math.sin(f * x)) < 1e-12
    # d/d dist and d/d freq of sum_k w_k rbf_k against the written-out derivatives
    w = torch.linspace(0.5, 2.0, r, dtype=torch.float64)
    g_dist, g_freq = torch.autograd.grad((rbf * w).sum(), [dist, layer.freq])
    want_gd, want_gf = [], [0.0] * r
    for d in dist.tolist():
        x = d / cutoff
        e, de = _env(x, expo)
        gd = 0.0
        for k in range(r):
            f = fr[k]
            gd += float(w[k]) * (de * math.sin(f * x) + e * f * math.cos(f * x)) / cutoff
            want_gf[k] += float(w[k]) * e * x * math.cos(f * x)
        want_gd.append(gd)
    torch.testing.assert_close(g_dist, torch.tensor(want_gd, dtype=torch.float64), rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(g_freq, torch.tensor(want_gf, dtype=torch.float64), rtol=1e-10, atol=1e-12)


def _create(c, use_gpu=False):
    import hydragnn_b200 as hb
    cfg = c["cfg"]
    return hb.create_model(mpnn_type="PNAPlus", input_dim=cfg["input_dim"], hidden_dim=cfg["hidden_dim"], output_dim=cfg["output_dim"],
                           output_type=cfg["output_type"], output_heads=cfg["output_heads"], activation_function="relu",
                           loss_function_type="mse", task_weights=[1.0] * len(cfg["output_type"]),
                           num_conv_layers=cfg["num_conv_layers"], edge_dim=cfg["edge_dim"], pna_deg=c["deg"],
                           graph_pooling=cfg["graph_pooling"], num_radial=cfg["num_radial"], radius=cfg["radius"],
                           envelope_exponent=cfg["envelope_exponent"], pe_dim=4 if cfg["gps"] else 0,
                           global_attn_engine="GPS" if cfg["gps"] else None, global_attn_type="multihead" if cfg["gps"] else None,
                           global_attn_heads=4 if cfg["gps"] else 0, use_gpu=use_gpu)


@pytest.mark.parametrize("name", CASES + ["pnaplus_mlip"])
def test_engine_pnaplus_stack_reproduces_the_reference_seeded_state(golden_dir, name):
    from hydragnn_b200.pnaplus import PNAPlusStack
    c = torch.load(golden_dir + "/models_pnaplus.pt")[name]
    m = _create(c)
    assert isinstance(m, PNAPlusStack) and str(m) == c["str"] == "PNAStack"
    assert list(m.state_dict().keys())[-1] == "rbf.freq"
    check_seeded_state(m, c["state"])


@pytest.mark.parametrize("name", ["pnaplus_graph_noedge", "pnaplus_node_edge_len", "pnaplus_multihead_h5", "pnaplus_edge_dim0",
                                  "pnaplus_add_pool_edge3"])
def test_oracle_stack_matches_reference_golden(golden_dir, name):
    """The oracle's whole PNAPlus stack (fp64) against the reference's PNAPlusStack.py + Base.py: eval and train-mode predictions,
    the loss, every parameter gradient (None where the reference's is None) and the BatchNorm running statistics."""
    c = torch.load(golden_dir + "/models_pnaplus.pt")[name]
    pos, ei = c["inputs"]["pos"], c["inputs"]["edge_index"]
    dist = (pos[ei[1]] - pos[ei[0]]).norm(dim=-1)
    assert float(dist.max()) > c["cfg"]["radius"] > float(dist.min())                    # edges on both sides of the cutoff
    check_golden_case(oracle_from_case("PNAPlus", c), c, lambda: golden_data(c["inputs"]), pred=(1e-6, 1e-5),
                      loss=(1e-6, 0), grads=grad_close(1e-4, 1e-6))


def test_edge_dim0_keeps_an_unused_edge_encoder(golden_dir):
    c = torch.load(golden_dir + "/models_pnaplus.pt")["pnaplus_edge_dim0"]
    enc = [k for k in c["state"] if "edge_encoder" in k]
    assert enc and all(c["grads"][k] is None for k in enc)
    assert c["state"]["graph_convs.0.module_0.edge_encoder.weight"].shape == (2, 2)      # Linear(F_in + 0, F_in)


def test_oracle_mlip_matches_reference_golden(golden_dir):
    """Energy + per-atom energy + force loss in eval mode: forces and the second-order parameter gradients."""
    c = torch.load(golden_dir + "/models_pnaplus.pt")["pnaplus_mlip"]
    m = oracle_from_case("PNAPlus", c)
    m.eval()
    d = golden_data(c["inputs"])
    d.pos.requires_grad_(True)
    pred = m(d)[0]
    g = int(d.batch.max()) + 1
    e = torch.zeros(g, dtype=torch.float64).index_add_(0, d.batch, pred[:, 0])
    forces = -torch.autograd.grad(e.sum(), d.pos, create_graph=True)[0]
    torch.testing.assert_close(forces.detach(), c["forces"].double(), rtol=1e-5, atol=1e-6)
    natoms = torch.bincount(d.batch).double()
    ee = torch.nn.functional.mse_loss(e, d.energy.double())
    ep = torch.nn.functional.mse_loss(e / natoms, d.energy.double() / natoms)
    ef = torch.nn.functional.mse_loss(forces, d.forces.double())
    tot = ee + ep + ef
    torch.testing.assert_close(float(tot), float(c["loss"]), rtol=1e-6, atol=0)
    grads = torch.autograd.grad(tot, list(m.parameters()), allow_unused=True)
    check_grads(c, {n: gr for (n, _), gr in zip(m.named_parameters(), grads)}, grad_close(1e-4, 1e-6))
