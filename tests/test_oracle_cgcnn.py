"""CGCNN on the CPU: the CGConv restatement (oracle/cgcnn.py) by hand-computed cases, the oracle stack against the
reference's own CGCNNStack.py + Base.py + gps.py (tests/golden/models_cgcnn.pt), and the engine's construction: seeded state
dict, names, ``str``, strict loading of the reference's checkpoint, and the refusals the reference shares."""
import math

import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import padded
from hydragnn_b200.cgcnn import CGCNNStack
from oracle.base import oracle_from_case
from oracle.cgcnn import CGCNNStackOracle, CGConv
from stack_support import check_golden_case, check_seeded_state, engine_kwargs, golden_data, grad_close

CASES = ["cgcnn_graph_edge0", "cgcnn_node_edge_len", "cgcnn_add_pool_edge3", "cgcnn_multihead", "cgcnn_mlp_per_node", "cgcnn_gps",
         "cgcnn_gps_edge2", "cgcnn_ci_width1"]


def _golden(golden_dir):
    return torch.load(golden_dir + "/models_cgcnn.pt")


def _sigmoid(v):
    return 1.0 / (1.0 + math.exp(-v))


def _softplus(v):
    return v if v > 20.0 else math.log1p(math.exp(v))


def _conv(dim, wf, bf, ws, bs):
    c = CGConv(1, dim).double()
    with torch.no_grad():
        c.lin_f.weight.copy_(torch.tensor([wf]))
        c.lin_f.bias.fill_(bf)
        c.lin_s.weight.copy_(torch.tensor([ws]))
        c.lin_s.bias.fill_(bs)
    return c


def test_cgconv_without_edge_attributes_by_hand():
    """z = [x_i | x_j] with x_i the target; node 0 receives nothing, so its output is x_0; node 2 sums two messages."""
    c = _conv(0, [0.5, -1.25], 0.1, [2.0, 0.75], -0.3)
    x = torch.tensor([[1.5], [-0.5], [0.25]], dtype=torch.float64)
    ei = torch.tensor([[0, 1, 0], [1, 2, 2]])
    out = c(x, ei)

    def m(xi, xj):
        return _sigmoid(0.5 * xi - 1.25 * xj + 0.1) * _softplus(2.0 * xi + 0.75 * xj - 0.3)
    want = [1.5, -0.5 + m(-0.5, 1.5), 0.25 + m(0.25, -0.5) + m(0.25, 1.5)]
    torch.testing.assert_close(out[:, 0], torch.tensor(want, dtype=torch.float64), rtol=1e-14, atol=0)


def test_cgconv_with_edge_attributes_by_hand():
    c = _conv(2, [0.5, -1.0, 0.25, -2.0], 0.2, [1.0, 0.5, -0.75, 1.5], 0.1)
    x = torch.tensor([[0.3], [-1.2]], dtype=torch.float64)
    ei = torch.tensor([[1, 0], [0, 1]])
    a = torch.tensor([[0.7, -0.4], [1.1, 0.9]], dtype=torch.float64)
    out = c(x, ei, a)

    def m(xi, xj, e):
        return (_sigmoid(0.5 * xi - 1.0 * xj + 0.25 * e[0] - 2.0 * e[1] + 0.2) *
                _softplus(1.0 * xi + 0.5 * xj - 0.75 * e[0] + 1.5 * e[1] + 0.1))
    want = [0.3 + m(0.3, -1.2, [0.7, -0.4]), -1.2 + m(-1.2, 0.3, [1.1, 0.9])]
    torch.testing.assert_close(out[:, 0], torch.tensor(want, dtype=torch.float64), rtol=1e-14, atol=0)


def test_cgconv_softplus_linear_branch_and_its_gradient():
    """A pre-activation s above 20 takes softplus's linear branch (torch's threshold): m = sigmoid(f) * s, dm/db_s = sigmoid(f),
    dm/db_f = s sigmoid(f) (1 - sigmoid(f))."""
    c = _conv(0, [0.5, 0.0], -0.2, [1.0, 0.0], 22.0)
    x = torch.tensor([[0.0], [1.0]], dtype=torch.float64)
    out = c(x, torch.tensor([[0], [1]]))
    f, s = 0.5 - 0.2, 1.0 + 22.0
    sg = _sigmoid(f)
    assert float(out[1, 0].detach()) == pytest.approx(1.0 + sg * s, rel=1e-15)
    gbf, gbs = torch.autograd.grad(out[1, 0], [c.lin_f.bias, c.lin_s.bias])
    assert float(gbs) == pytest.approx(sg, rel=1e-15)
    assert float(gbf) == pytest.approx(s * sg * (1 - sg), rel=1e-14)


@pytest.mark.parametrize("name", CASES)
def test_oracle_stack_matches_reference_golden(golden_dir, name):
    """The oracle's whole CGCNN stack (fp64) against the reference's: eval and train-mode predictions, the loss, every parameter
    gradient and the BatchNorm running statistics."""
    c = _golden(golden_dir)[name]
    check_golden_case(oracle_from_case(CGCNNStackOracle, c), c, lambda: golden_data(c["inputs"]), pred=(1e-6, 1e-5), loss=(1e-6, 0),
                      grads=grad_close(1e-4, 1e-6))


def engine_from_case(c, **kw):
    return hb.create_model(**engine_kwargs("CGCNN", c), use_gpu=False, **kw)


@pytest.mark.parametrize("name", CASES)
def test_engine_state_dict_and_str_match_the_reference(golden_dir, name):
    """Seeded construction: the engine's parameter and buffer names, order, shapes and values equal the reference's, and the
    reference's checkpoint loads strictly."""
    c = _golden(golden_dir)[name]
    eng = engine_from_case(c)
    assert isinstance(eng, CGCNNStack) and str(eng) == c["str"] == "CGCNNStack"
    check_seeded_state(eng, c["state"])
    assert all(isinstance(f.module, torch.nn.BatchNorm1d) for f in eng.feature_layers)


@pytest.mark.parametrize("key", ["conv_branch", "conv_legacy"])
def test_conv_node_heads_fail_as_the_reference_does(golden_dir, key):
    """CGCNN builds no conv-type node heads: the reference raises its ValueError for a branch whose "type" is "conv" and fails
    reading the branch's num_headlayers otherwise; the engine raises the same exception with the same message."""
    err = _golden(golden_dir)["errors"][key]
    assert err is not None
    kw = dict(input_dim=3, hidden_dim=3, output_dim=[1], output_type=["node"], output_heads=err["heads"], edge_dim=0, use_gpu=False)
    with pytest.raises(Exception) as info:
        hb.create_model(mpnn_type="CGCNN", **kw)
    assert type(info.value).__name__ == err["type"] and str(info.value) == err["msg"]


def test_missing_edge_attr_raises(golden_dir):
    from hydragnn_b200.cgcnn import CGConv as EngineCGConv
    conv = EngineCGConv(4, 2)
    with pytest.raises(ValueError, match="without edge_attr"):
        conv(torch.zeros(3, 4), None, None)


def test_edge_dim_none_without_gps_is_refused_at_construction(golden_dir):
    c = _golden(golden_dir)["cgcnn_graph_edge0"]
    with pytest.raises(ValueError, match="integer edge_dim"):
        engine_from_case(dict(c, cfg=dict(c["cfg"], edge_dim=None)))
    # under GPS the conv's edge input is the positional embedding, so edge_dim=None builds, as in the reference
    g = _golden(golden_dir)["cgcnn_gps"]
    assert isinstance(engine_from_case(dict(g, cfg=dict(g["cfg"], edge_dim=None))), CGCNNStack)


def test_hidden_dim_other_than_input_dim_without_gps_is_refused_before_any_launch(golden_dir):
    """The reference builds convs at input_dim behind BatchNorm(hidden_dim) and fails at the first BatchNorm; the engine builds
    the same modules and raises at forward, before touching the data."""
    c = _golden(golden_dir)["cgcnn_graph_edge0"]
    eng = engine_from_case(dict(c, cfg=dict(c["cfg"], hidden_dim=5)))
    assert eng.graph_convs[0].module_0.channels == 3 and eng.feature_layers[0].module.num_features == 5
    with pytest.raises(ValueError, match="hidden_dim is 5"):
        eng(golden_data(c["inputs"], torch.float32))


def test_padded_step_refuses_cgcnn(golden_dir):
    """BatchNorm feature layers: hb.train runs CGCNN stacks eagerly."""
    for name in ("cgcnn_graph_edge0", "cgcnn_ci_width1"):
        assert not padded.supported(engine_from_case(_golden(golden_dir)[name]))
