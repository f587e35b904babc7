"""CPU checks of activation_function "prelu" against tests/golden/models_prelu.pt, the reference's own Base.py, stacks and MACE
blocks run with one shared ``nn.PReLU()``: the fp64 oracle against the stack cases, the engine's seeded construction (names,
order, values, one slope tensor behind every alias), strict loads, ``str``, ``create_model_config``, and the ATen path
``ops.prelu`` takes for CPU tensors and any-order use."""
import pytest
import torch
from torch import nn

import hydragnn_b200 as hb
from hydragnn_b200 import ops
from hydragnn_b200.stacks import activation_function_selection
from oracle.base import oracle_from_case
from stack_support import (PRELU_CASES, PRELU_MACE_CASES, Flat, case_mpnn_type, check_golden_case, check_seeded_state, golden_data,
                           grad_close, named_case_kwargs, prelu_engine)

@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(golden_dir + "/models_prelu.pt")


@pytest.mark.parametrize("name", [n for n in PRELU_CASES if n != "pna_gps"])
def test_oracle_matches_reference_golden(golden, name):
    """The fp64 oracle against the reference: predictions, loss, every gradient (the shared slope's included, summed over every
    site) and the BatchNorm statistics.  (pna_gps runs the reference's gps.py, which the oracle does not restate.)"""
    c = golden[name]
    m = oracle_from_case(case_mpnn_type(name), c)
    # the reference names the shared slope where named_parameters first meets it, inside the first head; the oracle registers it
    # on the model first: its gradient is the same sum over every site under another name
    own = dict(m.named_parameters())
    name_of = {k: ("activation_function.weight" if k not in own else k) for k in c["grads"]}
    assert sum(k != v for k, v in name_of.items()) <= 1
    c = dict(c, grads={name_of[k]: g for k, g in c["grads"].items()})
    if c["cfg"].get("loss_function_type") == "GaussianNLLLoss":
        m = Flat(m)
    # the conv head's BatchNorm cancels the gradient of the bias before it, which the fp32 reference leaves at rounding level
    tol = grad_close(1e-3, 3e-5) if name == "pna_conv_head_slope" else grad_close(1e-4, 1e-6)
    check_golden_case(m, c, lambda: golden_data(c["inputs"]), pred=(1e-6, 1e-5), loss=(1e-6, 0), grads=tol)


@pytest.mark.parametrize("name", PRELU_CASES + ["mace"])
def test_engine_reproduces_the_reference_seeded_state(golden, name):
    """Names, order and values of the engine's seeded state dict equal the reference's, every alias of the one slope included;
    the reference's state loads strictly and comes back unchanged."""
    c = golden[name]
    m = prelu_engine(name, c)
    assert list(m.state_dict()) == c["keys"]
    if name != "mace":
        check_seeded_state(m, c["state"])
        return
    params = dict(m.named_parameters())                 # MACE's coupling buffers are computed, equal to rounding
    for k, v in m.state_dict().items():
        assert torch.equal(v, c["state"][k]) if k in params else torch.allclose(v, c["state"][k], atol=1e-6), k
    m.load_state_dict(c["state"], strict=True)


def test_mace_film_keys_after_the_conditioner_exists(golden):
    """FiLM's graph_conditioner (created at the first forward) holds the shared PReLU: the reference lists it there, after every
    other entry.  The engine builds the same conditioner: its entries come in the same order and hold the same slope tensor."""
    c = golden["mace_film"]
    m = prelu_engine("mace_film", c)
    m._ensure_graph_conditioner(2, torch.device("cpu"))
    assert list(m.state_dict()) == c["keys"]
    assert m.graph_conditioner[1] is m.activation_function


@pytest.mark.parametrize("name", PRELU_CASES + PRELU_MACE_CASES)
def test_one_slope_tensor_behind_every_alias(golden, name):
    c = golden[name]
    m = prelu_engine(name, c)
    if name == "mace_film":
        m._ensure_graph_conditioner(2, torch.device("cpu"))
    sd = m.state_dict(keep_vars=True)
    slope = c["state"]["activation_function.weight"]
    aliases = [k for k in c["keys"] if k.endswith(".weight") and c["state"][k].shape == (1,) and torch.equal(c["state"][k], slope)]
    assert "activation_function.weight" in aliases
    for k in aliases:
        assert sd[k] is m.activation_function.weight, k
    assert sum(p is m.activation_function.weight for p in m.parameters()) == 1     # the optimiser sees one slope


def test_no_reference_refusals(golden):
    assert golden["errors"] == {}


@pytest.mark.parametrize("name", PRELU_CASES + ["mace"])
def test_str_and_strict_loads_both_ways(golden, name):
    c = golden[name]
    m = prelu_engine(name, c)
    relu = hb.create_model(**dict(named_case_kwargs(name, c), activation_function="relu"), use_gpu=False)
    assert str(m) == str(relu)
    m.load_state_dict(c["state"], strict=True)
    sd = m.state_dict()
    fresh = prelu_engine(name, c)
    fresh.load_state_dict(sd, strict=True)
    assert all(torch.equal(v, fresh.state_dict()[k]) for k, v in sd.items())


@pytest.mark.parametrize("mpnn", ["PNA", "EGNN", "PAINN", "SAGE", "MFC", "CGCNN", "GAT", "PNAPlus", "PNAEq", "SchNet"])
def test_create_model_config_builds_every_stack_with_prelu(mpnn):
    arch = {"mpnn_type": mpnn, "input_dim": 3, "hidden_dim": 8, "num_conv_layers": 2, "pna_deg": [0, 2, 3], "edge_dim": None,
            "num_radial": 5, "radius": 5.0, "max_neighbours": 5, "num_gaussians": 10, "num_filters": 8,
            "output_heads": {"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 10, "num_headlayers": 2, "dim_headlayers": [10, 10]}},
            "output_dim": [1], "output_type": ["graph"], "task_weights": [1.0], "activation_function": "prelu"}
    if mpnn == "PNAPlus":
        arch.update(envelope_exponent=5)
    if mpnn == "CGCNN":
        arch.update(edge_dim=0, hidden_dim=3)
    m = hb.create_model_config({"Architecture": arch, "Training": {"loss_function_type": "mse"}}, use_gpu=False)
    assert isinstance(m.activation_function, nn.PReLU)
    shared = m.graph_shared["branch-0"]
    assert shared[1] is m.activation_function and m.heads_NN[0]["branch-0"][1] is m.activation_function
    assert float(m.activation_function.weight.detach()) == 0.25


def test_activation_selection():
    a = activation_function_selection("prelu")
    assert type(a) is nn.PReLU and a.weight.shape == (1,) and float(a.weight) == 0.25
    for name in ("relu", "selu", "elu", "sigmoid", "lrelu_01", "lrelu_025", "lrelu_05"):
        assert not isinstance(activation_function_selection(name), nn.PReLU)
    with pytest.raises(ValueError, match="Unknown activation"):
        activation_function_selection("gelu")


@pytest.mark.parametrize("slope", [0.25, 0.0, -0.7])
def test_prelu_cpu_and_any_order_path_is_atens(slope):
    """``ops.prelu`` on CPU tensors or with higher_order is ``F.prelu``: value, first and second gradients."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(50, 7, generator=g, dtype=torch.float64)
    x[0, :3] = 0.0
    w = torch.tensor([slope], dtype=torch.float64)
    for higher in (False, True):
        xa, wa = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        xb, wb = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        ya, yb = ops.prelu(xa, wa, higher), torch.nn.functional.prelu(xb, wb)
        assert torch.equal(ya, yb)
        ga = torch.autograd.grad((ya * ya).sum(), (xa, wa), create_graph=True)
        gb = torch.autograd.grad((yb * yb).sum(), (xb, wb), create_graph=True)
        for p, q in zip(ga, gb):
            assert torch.equal(p, q)
