"""CPU checks of GaussianNLLLoss (mean-and-variance heads) against tests/golden/models_gnll.pt, the reference's own Base.py and
stack files run with loss_function_type "GaussianNLLLoss": the fp64 oracle against every case, the engine's seeded construction,
``var_output`` / ``str`` / the ``create_model_config`` path, the refusals, and the any-order ATen NLL against torch's own."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import ops
from oracle.base import oracle_from_case
from stack_support import (GNLL_CASES, Flat, case_mpnn_type, check_golden_case, check_seeded_state, golden_data, grad_close,
                           named_case_kwargs)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir + "/models_gnll.pt")


@pytest.mark.parametrize("name", [n for n in GNLL_CASES if n != "pna_gps"])
def test_oracle_matches_reference_golden(golden, name):
    """The fp64 oracle against the reference: eval and train-mode means and variances, the NLL, every parameter gradient and the
    BatchNorm statistics after the step.  (pna_gps runs the reference's gps.py, which the oracle does not restate.)"""
    c = golden[name]
    # the conv head ends in BatchNorm + ReLU, so about half its variances are exactly 0 and clamped to eps: the fp32 reference's
    # gradients then carry terms of (mean - target) / eps, and their rounding sets the bound
    atol = 1e-5 if name == "pna_conv_head" else 1e-6
    check_golden_case(Flat(oracle_from_case(case_mpnn_type(name), c)), c, lambda: golden_data(c["inputs"]), pred=(1e-6, 1e-5),
                      loss=(1e-6, 0), grads=grad_close(1e-4, atol))


@pytest.mark.parametrize("name", [n for n in GNLL_CASES if n != "egnn_clamped"])
def test_engine_reproduces_the_reference_seeded_state(golden, name):
    """Head widths doubled at every site (graph heads, mlp / mlp_per_node, conv heads and their BatchNorms), initial_bias over
    all 2 d entries: the engine's seeded state dict equals the reference's key for key and value for value."""
    c = golden[name]
    m = hb.create_model(**named_case_kwargs(name, c), use_gpu=False)
    assert m.var_output == 1 and m.loss_function_type == "GaussianNLLLoss"
    check_seeded_state(m, c["state"])


def test_str_var_output_and_create_model_config():
    cfg = {"Architecture": {"mpnn_type": "PNA", "input_dim": 1, "hidden_dim": 8, "num_conv_layers": 2, "pna_deg": [0, 2, 3],
                            "output_heads": {"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 10, "num_headlayers": 2,
                                                       "dim_headlayers": [10, 10]}},
                            "output_dim": [1], "output_type": ["graph"], "task_weights": [1.0]},
           "Training": {"loss_function_type": "GaussianNLLLoss"}}
    m = hb.create_model_config(cfg, use_gpu=False)
    assert m.var_output == 1 and str(m) == "PNAStack"
    assert m.heads_NN[0]["branch-0"][-1].out_features == 2
    mse = hb.create_model_config(dict(cfg, Training={"loss_function_type": "mse"}), use_gpu=False)
    assert mse.var_output == 0 and mse.heads_NN[0]["branch-0"][-1].out_features == 1


GRAPH = {"num_sharedlayers": 1, "dim_sharedlayers": 4, "num_headlayers": 1, "dim_headlayers": [4]}
CONV = {"num_headlayers": 2, "dim_headlayers": [10, 6], "type": "conv"}
MLP = {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}
REFUSED = {
    "mace": dict(mpnn_type="MACE", output_dim=[1, 1], output_type=["graph", "node"], output_heads={"graph": GRAPH, "node": MLP},
                 radius=6.0, num_radial=8, max_ell=2, node_max_ell=1, avg_num_neighbors=10.0, num_nodes=9),
    "mlip": dict(mpnn_type="EGNN", output_dim=[1], output_type=["node"], output_heads={"node": MLP}, enable_interatomic_potential=True,
                 energy_weight=1.0, force_weight=1.0),
    "gat_conv_head": dict(mpnn_type="GAT", output_dim=[1], output_type=["node"], output_heads={"node": CONV}),
    "cgcnn_conv_head": dict(mpnn_type="CGCNN", hidden_dim=3, edge_dim=0, output_dim=[1], output_type=["node"],
                            output_heads={"node": CONV}),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refusals(golden, name):
    """What the reference cannot run under GaussianNLLLoss is refused at construction, before any launch.  The reference fails
    later and in its own way: MACE's loss unpacks the output list as (pred, var), the MLIP loss reads pred[0] as a tensor, GAT's
    node convs give a [N, 0] variance that torch's GaussianNLLLoss rejects with a ValueError.  Its CGCNN conv-type node heads
    fail at construction whatever the loss, with the KeyError the engine raises too."""
    ref = golden["errors"][name]
    kw = dict(dict(input_dim=3, hidden_dim=8, activation_function="relu", loss_function_type="GaussianNLLLoss", use_gpu=False),
              **REFUSED[name])
    want = KeyError if ref["type"] == "KeyError" else ValueError
    with pytest.raises(want) as e:
        hb.create_model(**kw)
    if name == "gat_conv_head":
        assert ref["type"] == "ValueError" and ref["msg"] == "var is of incorrect size"
    if want is ValueError:
        assert "GaussianNLLLoss is not supported" in str(e.value)
    kw["loss_function_type"] = "mse"                               # the same models build under mse (CGCNN's conv heads excepted)
    if name != "cgcnn_conv_head":
        hb.create_model(**kw)


def _nll_inputs(n=64, d=3):
    g = torch.Generator().manual_seed(5)
    mean = torch.randn(n, d, generator=g, dtype=torch.float64)
    target = torch.randn(n, d, generator=g, dtype=torch.float64)
    s = torch.randn(n, d, generator=g, dtype=torch.float64)
    s[: n // 4] *= 1e-4                                             # var = s^2 below eps: clamped
    s[n // 4: n // 2] = 0.0
    return mean, target, s


@pytest.mark.parametrize("mask", [False, True])
def test_any_order_nll_matches_torch_on_both_sides_of_the_clamp(mask):
    """Value, first and second gradients of ``ops.gaussian_nll_any_order`` against torch.nn.functional.gaussian_nll_loss, with a
    quarter of the variances under eps, a quarter exactly zero; with a 0/1 mask, against torch's loss over the kept rows."""
    mean, target, s = _nll_inputs()
    keep = torch.arange(mean.shape[0]) < 40
    m = keep[:, None].to(mean.dtype).expand_as(mean)
    results = []
    for ours in (True, False):
        mu = mean.clone().requires_grad_(True)
        sv = s.clone().requires_grad_(True)
        var = sv * sv
        if ours:
            val = ops.gaussian_nll_any_order(mu, var, target, m, m.sum()) if mask else ops.gaussian_nll_any_order(mu, var, target)
        elif mask:
            val = torch.nn.functional.gaussian_nll_loss(mu[keep], target[keep], var[keep])
        else:
            val = torch.nn.functional.gaussian_nll_loss(mu, target, var)
        g_mu, g_s = torch.autograd.grad(val, (mu, sv), create_graph=True)
        hv = torch.autograd.grad((g_mu.sum() + g_s.sum()), (mu, sv))
        results.append([val.detach(), g_mu.detach(), g_s.detach(), *hv])
    for a, b in zip(*results):
        torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)


def test_loss_selection_keeps_mse_mae_rmse_and_names_the_choices():
    from hydragnn_b200.stacks import _Loss, loss_function_selection
    assert all(isinstance(loss_function_selection(n), _Loss) for n in ("mse", "mae", "rmse"))
    with pytest.raises(ValueError, match="GaussianNLLLoss"):
        loss_function_selection("smooth_l1")
