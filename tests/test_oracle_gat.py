"""GAT on the CPU: the GATv2Conv restatement (oracle/gat.py) by hand-computed cases, the oracle stack against the
reference's own GATStack.py + Base.py + gps.py (tests/golden/models_gat.pt), and the engine's construction: seeded state dict,
names, ``str``, strict loading of the reference's checkpoint, and the refusals."""
import math

import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import ops, padded
from hydragnn_b200.gat import GATStack
from oracle.base import oracle_from_case
from oracle.gat import GATStackOracle, GATv2Conv
from stack_support import check_golden_case, engine_kwargs, golden_data, grad_close, seeded_state, state_digest

CASES = ["gat_graph_noedge", "gat_node_edge_len", "gat_multihead", "gat_add_pool_edge3", "gat_one_layer", "gat_input_ne_hidden",
         "gat_conv_head", "gat_gps", "gat_gps_edge2", "gat_loops_dups_isolated"]


def _golden(golden_dir):
    return torch.load(golden_dir + "/models_gat.pt")


# ---- GATv2Conv by hand: 3 nodes, 2 heads, 1 channel per head -------------------------------------------------------------
# edges (src -> dst): 0 -> 1, 2 -> 1, 1 -> 1 (an input self-loop, removed), 1 -> 2; node 0 receives nothing but its self-loop.
EI = torch.tensor([[0, 2, 1, 1], [1, 1, 1, 2]])
EA = torch.tensor([[1.0], [3.0], [100.0], [-2.0]])         # the self-loop's 100 must not enter node 1's mean attribute
X = torch.tensor([[1.0], [-2.0], [0.5]])
SLOPE = 0.05


def _hand_conv(concat, with_edge):
    c = GATv2Conv(1, 1, heads=2, concat=concat, negative_slope=SLOPE, edge_dim=1 if with_edge else None).double()
    with torch.no_grad():
        c.lin_l.weight.copy_(torch.tensor([[1.0], [-1.0]], dtype=torch.float64))
        c.lin_l.bias.copy_(torch.tensor([0.5, 0.0], dtype=torch.float64))
        c.lin_r.weight.copy_(torch.tensor([[2.0], [0.5]], dtype=torch.float64))
        c.lin_r.bias.copy_(torch.tensor([-1.0, 0.25], dtype=torch.float64))
        c.att.copy_(torch.tensor([[[1.5], [-0.5]]], dtype=torch.float64))
        if with_edge:
            c.lin_edge.weight.copy_(torch.tensor([[0.3], [-0.2]], dtype=torch.float64))
        c.bias.copy_(torch.tensor([0.1, -0.2], dtype=torch.float64) if concat else torch.tensor([0.3], dtype=torch.float64))
    return c


def _hand_expected(concat, with_edge, x, ea):
    """The published algorithm as scalar loops (x, ea: lists of floats)."""
    wl, bl, wr, br, att = [1.0, -1.0], [0.5, 0.0], [2.0, 0.5], [-1.0, 0.25], [1.5, -0.5]
    we = [0.3, -0.2]
    edges = [(0, 1, ea[0]), (2, 1, ea[1]), (1, 2, ea[3])]                     # input self-loop 1 -> 1 removed
    mean = {}
    for i in range(3):
        a = [e[2] for e in edges if e[1] == i]
        mean[i] = sum(a) / len(a) if a else 0.0
    edges += [(i, i, mean[i]) for i in range(3)]
    out = []
    for i in range(3):
        per_head = []
        for h in range(2):
            sc = []
            for j, t, a in edges:
                if t != i:
                    continue
                z = (wr[h] * x[i] + br[h]) + (wl[h] * x[j] + bl[h]) + (we[h] * a if with_edge else 0.0)
                lr = z if z > 0 else SLOPE * z
                sc.append((lr * att[h], wl[h] * x[j] + bl[h]))
            m = max(s for s, _ in sc)
            den = sum(math.exp(s - m) for s, _ in sc) + 1e-16
            per_head.append(sum(math.exp(s - m) / den * v for s, v in sc))
        out.append([per_head[0] + 0.1, per_head[1] - 0.2] if concat else [(per_head[0] + per_head[1]) / 2 + 0.3])
    return torch.tensor(out, dtype=torch.float64)


@pytest.mark.parametrize("concat", [True, False])
@pytest.mark.parametrize("with_edge", [False, True])
def test_gatv2conv_hand_computed(concat, with_edge):
    c = _hand_conv(concat, with_edge)
    got = c(X.double(), EI, EA.double() if with_edge else None)
    want = _hand_expected(concat, with_edge, X[:, 0].tolist(), EA[:, 0].tolist())
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)
    # both leaky branches are taken: z of the edge 1 -> 2 is negative on head 0 and positive on head 1
    xl, xr = c.lin_l(X.double()), c.lin_r(X.double())
    z = xr[2] + xl[1]
    assert z[0] < 0 < z[1]


@pytest.mark.parametrize("concat", [True, False])
def test_gatv2conv_hand_computed_gradients(concat):
    """d out / d (x, edge_attr) of the restatement equals the gradient of the scalar-loop statement (central differences)."""
    c = _hand_conv(concat, True)
    x, ea = X.double().clone().requires_grad_(True), EA.double().clone().requires_grad_(True)
    wgt = torch.linspace(-1.0, 1.5, 6 if concat else 3, dtype=torch.float64).view(3, -1)
    gx, ge = torch.autograd.grad((c(x, EI, ea) * wgt).sum(), (x, ea))

    def f(xs, es):
        return float((_hand_expected(concat, True, xs, es) * wgt).sum())

    h = 1e-6
    for k in range(3):
        xp, xm = X[:, 0].tolist(), X[:, 0].tolist()
        xp[k] += h
        xm[k] -= h
        assert abs((f(xp, EA[:, 0].tolist()) - f(xm, EA[:, 0].tolist())) / (2 * h) - float(gx[k, 0])) < 1e-7
    for k in range(4):
        ep, em = EA[:, 0].tolist(), EA[:, 0].tolist()
        ep[k] += h
        em[k] -= h
        assert abs((f(X[:, 0].tolist(), ep) - f(X[:, 0].tolist(), em)) / (2 * h) - float(ge[k, 0])) < 1e-7
    assert float(ge[2, 0]) == 0.0                                  # the removed input self-loop's attribute is unused


@pytest.mark.parametrize("name", CASES)
def test_oracle_stack_matches_reference_golden(golden_dir, name):
    c = _golden(golden_dir)[name]
    # the golden is the reference's fp32 arithmetic: the 120-wide head convs of gat_conv_head put its loss 1.2e-6 from fp64, and a
    # conv bias in front of a BatchNorm, which has no gradient in exact arithmetic, holds up to 1.1e-6 gmax there
    check_golden_case(oracle_from_case(GATStackOracle, c, seeded_state(c)), c, lambda: golden_data(c["inputs"]), pred=(1e-6, 1e-5),
                      loss=(5e-6, 0), grads=grad_close(1e-4, 2e-6))


def engine_from_case(c, **kw):
    return hb.create_model(**engine_kwargs("GAT", c), use_gpu=False, **kw)


@pytest.mark.parametrize("name", CASES)
def test_engine_state_dict_and_str_match_the_reference(golden_dir, name):
    """Seeded construction: the engine's parameter and buffer names, order, shapes and values equal the reference's, and the
    reference's checkpoint loads strictly.  The stack-level out_lin the reference assigns in get_conv is parameter-free."""
    c = _golden(golden_dir)[name]
    eng = engine_from_case(c)
    assert isinstance(eng, GATStack) and str(eng) == c["str"] == "GATStack"
    want, se = c["state_sha256"], eng.state_dict()
    assert list(want.keys()) == list(se.keys())
    for k in want:
        assert state_digest(se[k]) == want[k], k
    sr = seeded_state(c)
    eng.load_state_dict(sr, strict=True)
    assert not any(k.startswith("out_lin") for k in se) and "out_lin" in c["top_level"]
    assert isinstance(eng.out_lin, torch.nn.Identity)


def test_one_conv_layer_builds_two_convs(golden_dir):
    eng = engine_from_case(_golden(golden_dir)["gat_one_layer"])
    assert len(eng.graph_convs) == len(eng.feature_layers) == 2
    assert eng.graph_convs[0].module_0.concat and not eng.graph_convs[1].module_0.concat
    assert eng.feature_layers[0].module.num_features == 4 * 6 and eng.feature_layers[1].module.num_features == 4


def test_conv_head_with_edge_features_fails_as_the_reference_does(golden_dir):
    """The reference's head convs have no lin_edge and PyG's GATv2Conv asserts when handed edge_attr; the engine raises the same
    exception type before touching the data."""
    err = _golden(golden_dir)["errors"]["conv_head_edge_attr"]
    assert err["type"] == "AssertionError"
    heads = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [20, 10], "type": "conv"}}]}
    eng = hb.create_model(mpnn_type="GAT", input_dim=1, hidden_dim=4, output_dim=[1], output_type=["node"], output_heads=heads,
                          edge_dim=1, num_conv_layers=2, use_gpu=False)
    c = _golden(golden_dir)["gat_node_edge_len"]
    with pytest.raises(AssertionError):
        eng(golden_data(c["inputs"], torch.float32))


def test_existing_refusals_stay():
    conv = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 1, "dim_headlayers": [4], "type": "conv"}}]}
    with pytest.raises(ValueError, match="without global attention"):
        hb.create_model(mpnn_type="GAT", input_dim=2, hidden_dim=4, output_dim=[1], output_type=["node"], output_heads=conv,
                        pe_dim=4, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=2, use_gpu=False)
    with pytest.raises(ValueError, match="edge_dim None"):
        hb.create_model(mpnn_type="GAT", input_dim=2, hidden_dim=4, output_dim=[1], output_type=["graph"], edge_dim=0,
                        output_heads={"graph": {"num_sharedlayers": 1, "dim_sharedlayers": 4, "num_headlayers": 1,
                                                "dim_headlayers": [4]}}, use_gpu=False)


def test_engine_conv_raises_pyg_assertion_for_edge_attr_without_lin_edge():
    from hydragnn_b200.gat import GATv2Conv as EngineConv
    conv = EngineConv(4, 2, heads=3)
    with pytest.raises(AssertionError):
        conv(torch.zeros(3, 4), None, (torch.zeros(2, 1), None))


def test_kernel_shape_limits():
    """hgb_gat_supported: 1 <= heads <= 8, heads c <= 512 with c a multiple of 4 (256 otherwise), 0 <= d <= 16."""
    assert ops.gat_supported(6, 64, 1) and ops.gat_supported(8, 64, 16) and ops.gat_supported(1, 1, 0)
    assert ops.gat_supported(8, 32, 0) and ops.gat_supported(6, 20, 7) and not ops.gat_supported(6, 128, 0)
    assert ops.gat_supported(8, 31, 0) and not ops.gat_supported(8, 33, 0)
    assert not ops.gat_supported(9, 1, 0) and not ops.gat_supported(0, 4, 0) and not ops.gat_supported(6, 4, 17)


def test_padded_step_refuses_gat(golden_dir):
    """BatchNorm feature layers: hb.train runs GAT stacks eagerly."""
    for name in ("gat_graph_noedge", "gat_add_pool_edge3"):
        assert not padded.supported(engine_from_case(_golden(golden_dir)[name]))
