"""CPU checks of the PNAConv restatement (oracle/pna.py) and of the engine's seeded construction.

models_pna.pt pins the reference's PNAStack / Base code with this restatement standing in for PyG's PNAConv, so the
restatement itself is pinned here by hand-computed cases: x_i (the target, edge_index[1]) is the first block of the pre_nn
input, the four aggregators with an empty segment (zeros), a single edge (std masked to 0), a tie, and an edge attribute.
"""
import math

import pytest
import torch

from hydragnn_b200.pna import AGGREGATORS, SCALERS, PNAStack
from oracle.base import oracle_from_case
from oracle.pna import PNAConv
from stack_support import check_golden_case, check_seeded_state, golden_data, grad_close

# nodes 0..4, x = [1, 2, 4, 8, 16]; edges (source -> target): 1->0, 2->0 (two into 0), 0->3 (one), 2->4 twice (a tie);
# nodes 1 and 2 receive nothing
X = torch.tensor([[1.0], [2.0], [4.0], [8.0], [16.0]], dtype=torch.float64)
EI = torch.tensor([[1, 2, 0, 2, 2], [0, 0, 3, 4, 4]])
DEG_HIST = [2.0, 1.0, 2.0]                    # two nodes of in-degree 0, one of 1, two of 2


def _conv(edge_dim=None):
    conv = PNAConv(1, 17, AGGREGATORS, SCALERS, torch.tensor(DEG_HIST), edge_dim=edge_dim).double()
    with torch.no_grad():
        pre = conv.pre_nns[0][0]
        pre.weight.copy_(torch.tensor([[1.0, 10.0] + ([1.0] if edge_dim else [])]))     # h = x_i + 10 x_j (+ enc)
        pre.bias.zero_()
        post = conv.post_nns[0][0]
        post.weight.copy_(torch.eye(17))                                                 # the 17 post inputs, unchanged
        post.bias.zero_()
        conv.lin.weight.copy_(torch.eye(17))
        conv.lin.bias.zero_()
        if edge_dim:
            conv.edge_encoder.weight.fill_(2.0)
            conv.edge_encoder.bias.fill_(1.0)                                             # enc = 2 a + 1
    return conv


def _expected(h_by_node):
    """[x | A | A amp | A att | A lin] with A = [mean, min, max, std] per node, written out from the definitions."""
    avg_lin = (0 * 2 + 1 * 1 + 2 * 2) / 5.0
    avg_log = (math.log(1) * 2 + math.log(2) * 1 + math.log(3) * 2) / 5.0
    avg_lin, avg_log = float(torch.tensor(avg_lin, dtype=torch.float32)), float(torch.tensor(avg_log, dtype=torch.float32))
    rows = []
    for i, hs in enumerate(h_by_node):
        if hs:
            mean = sum(hs) / len(hs)
            var = sum(v * v for v in hs) / len(hs) - mean * mean
            std = math.sqrt(max(var, 1e-5))
            std = 0.0 if std <= math.sqrt(1e-5) else std
            a = [mean, min(hs), max(hs), std]
        else:
            a = [0.0] * 4
        d = max(len(hs), 1)
        amp, att, lin = math.log(d + 1) / avg_log, avg_log / math.log(d + 1), d / avg_lin
        rows.append([float(X[i, 0])] + a + [v * amp for v in a] + [v * att for v in a] + [v * lin for v in a])
    return torch.tensor(rows, dtype=torch.float64)


def test_pna_conv_hand_computed_without_edge_attributes():
    # target first: 1->0 gives 1 + 10*2 = 21, 2->0 gives 1 + 40 = 41 (mean 31, std 10); 0->3 gives 8 + 10 = 18 (one edge:
    # std masked); 2->4 twice gives 56, 56 (a tie, std 0); nodes 1 and 2 are empty segments
    out = _conv()(X, EI).detach()
    want = _expected([[21.0, 41.0], [], [], [18.0], [56.0, 56.0]])
    torch.testing.assert_close(out.detach(), want, rtol=1e-12, atol=1e-12)
    assert float(out[0, 4]) == 10.0 and float(out[3, 4]) == 0.0 and float(out[4, 4]) == 0.0
    assert torch.all(out[1:3, 1:] == 0)


def test_pna_conv_hand_computed_with_an_edge_attribute():
    a = torch.tensor([[0.5], [-1.0], [2.0], [0.0], [0.0]], dtype=torch.float64)      # enc = 2 a + 1 = [2, -1, 5, 1, 1]
    out = _conv(edge_dim=1)(X, EI, a)
    want = _expected([[23.0, 40.0], [], [], [23.0], [57.0, 57.0]])
    torch.testing.assert_close(out.detach(), want, rtol=1e-12, atol=1e-12)


def test_pna_conv_two_edges_into_one_node_width_one():
    # F_in = 1 end to end through real (seeded) post / lin Linears: the output is lin(post([x | scaled A])) by hand
    torch.manual_seed(3)
    conv = PNAConv(1, 3, AGGREGATORS, SCALERS, torch.tensor([0.0, 0.0, 1.0])).double()
    x = torch.tensor([[0.5], [1.5], [-2.0]], dtype=torch.float64)
    ei = torch.tensor([[1, 2], [0, 0]])
    w, b = conv.pre_nns[0][0].weight[0], conv.pre_nns[0][0].bias[0]
    h = [float(w[0] * x[0, 0] + w[1] * x[1, 0] + b), float(w[0] * x[0, 0] + w[1] * x[2, 0] + b)]
    mean = sum(h) / 2
    std = math.sqrt(max((h[0] ** 2 + h[1] ** 2) / 2 - mean * mean, 1e-5))
    A = torch.tensor([mean, min(h), max(h), std], dtype=torch.float64)
    s = float(conv.aggr_module.avg_deg_log) / math.log(3)                          # avg_deg_log = log 3, deg 2
    feats = torch.cat([x[0], A, A * (1 / s), A * s, A * (2 / float(conv.aggr_module.avg_deg_lin))])
    want0 = conv.lin(conv.post_nns[0][0](feats))
    out = conv(x, ei)
    torch.testing.assert_close(out[0].detach(), want0.detach(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", ["pna_graph_noedge", "pna_node_edge_len", "pna_multihead_h5", "pna_gps", "pna_add_pool_edge3"])
def test_engine_pna_stack_reproduces_the_reference_seeded_state(golden_dir, name):
    import hydragnn_b200 as hb
    c = torch.load(golden_dir + "/models_pna.pt")[name]
    cfg = c["cfg"]
    m = hb.create_model(mpnn_type="PNA", input_dim=cfg["input_dim"], hidden_dim=cfg["hidden_dim"], output_dim=cfg["output_dim"],
                        output_type=cfg["output_type"], output_heads=cfg["output_heads"], activation_function="relu",
                        loss_function_type="mse", task_weights=[1.0] * len(cfg["output_type"]), num_conv_layers=cfg["num_conv_layers"],
                        edge_dim=cfg["edge_dim"], pna_deg=c["deg"], graph_pooling=cfg["graph_pooling"],
                        pe_dim=4 if cfg["gps"] else 0, global_attn_engine="GPS" if cfg["gps"] else None,
                        global_attn_type="multihead" if cfg["gps"] else None, global_attn_heads=4 if cfg["gps"] else 0, use_gpu=False)
    assert isinstance(m, PNAStack) and str(m) == "PNAStack"
    check_seeded_state(m, c["state"])


@pytest.mark.parametrize("name", ["pna_graph_noedge", "pna_node_edge_len", "pna_multihead_h5", "pna_add_pool_edge3"])
def test_oracle_stack_matches_reference_golden(golden_dir, name):
    """The oracle's whole PNA stack (fp64) against the reference's PNAStack.py + Base.py: eval and train-mode predictions, the loss,
    every parameter gradient and the BatchNorm running statistics after the step.  (GPS is the reference's gps.py, not restated.)"""
    c = torch.load(golden_dir + "/models_pna.pt")[name]
    check_golden_case(oracle_from_case("PNA", c), c, lambda: golden_data(c["inputs"]), pred=(1e-6, 1e-5), loss=(1e-6, 0),
                      grads=grad_close(1e-4, 1e-6))


def test_pna_conv_with_edge_dim_refuses_a_missing_edge_attr():
    # PyG feeds [x_i | x_j] (2F) to the 3F-wide pre_nn and fails; the engine must not silently drop the W_c columns instead
    from hydragnn_b200.pna import PNAConv as EnginePNAConv
    conv = EnginePNAConv(4, 4, AGGREGATORS, SCALERS, torch.tensor(DEG_HIST), edge_dim=1)
    with pytest.raises(ValueError, match="without edge_attr"):
        conv(torch.zeros(3, 4), None, None)
