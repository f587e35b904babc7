"""SAGE and MFC on the CPU: the SAGEConv / MFConv restatements (oracle/sage.py) by hand-computed cases, and the oracle stacks
against the reference's own SAGEStack.py / MFCStack.py + Base.py + gps.py (tests/golden/models_sage.pt, models_mfc.pt)."""
import pytest
import torch

from oracle.base import oracle_from_case
from oracle.sage import MFCStackOracle, MFConv, SAGEConv, SAGEStackOracle
from stack_support import check_golden_case, golden_data, grad_close

SAGE_CASES = ["sage_graph", "sage_node", "sage_multihead", "sage_mlp_per_node", "sage_conv_head", "sage_max_pool_in1", "sage_gps",
              "sage_initial_bias", "sage_initial_bias_node"]
MFC_CASES = ["mfc_graph_deg5", "mfc_node_deg1", "mfc_multihead_deg100", "mfc_mlp_per_node", "mfc_conv_head", "mfc_max_pool_in1",
             "mfc_gps", "mfc_initial_bias_node"]


def _set(lin, w, b=None):
    with torch.no_grad():
        lin.weight.copy_(torch.tensor(w, dtype=torch.float64))
        if b is not None:
            lin.bias.copy_(torch.tensor(b, dtype=torch.float64))


def test_sageconv_by_hand():
    """out_i = W_l mean_j x_j + b_l + W_r x_i; node 0 has no in-edges, so its mean is 0; node 2 has a duplicate edge."""
    c = SAGEConv(1, 1).double()
    _set(c.lin_l, [[2.0]], [0.5])
    _set(c.lin_r, [[-1.5]])
    x = torch.tensor([[1.0], [3.0], [-2.0]], dtype=torch.float64)
    ei = torch.tensor([[0, 1, 0, 0], [1, 2, 2, 2]])
    out = c(x, ei)[:, 0]
    want = [0.5 - 1.5 * 1.0, 2.0 * 1.0 + 0.5 - 1.5 * 3.0, 2.0 * (3.0 + 1.0 + 1.0) / 3 + 0.5 + 3.0]
    torch.testing.assert_close(out, torch.tensor(want, dtype=torch.float64), rtol=1e-15, atol=1e-15)


def test_mfconv_by_hand_degree_clamp_and_zero_gradients():
    """deg_i = min(in-degree, max_degree) counting duplicates and self-loops; degree-0 nodes use lins_l[0]; a degree no node has
    still gets a gradient, of zeros."""
    c = MFConv(1, 1, max_degree=2).double()
    for d in range(3):
        _set(c.lins_l[d], [[1.0 + d]], [10.0 * d])
        _set(c.lins_r[d], [[-(d + 0.5)]])
    x = torch.tensor([[1.0], [2.0], [4.0]], dtype=torch.float64)
    ei = torch.tensor([[0, 1, 2, 2], [2, 2, 2, 0]])           # node 2: three in-edges (one a self-loop) -> clamped to 2
    out = c(x, ei)[:, 0]
    want = [2.0 * 4.0 + 10.0 - 1.5 * 1.0,                     # node 0: degree 1
            1.0 * 0.0 + 0.0 - 0.5 * 2.0,                       # node 1: degree 0, h = 0
            3.0 * 7.0 + 20.0 - 2.5 * 4.0]                      # node 2: degree 3 -> 2
    torch.testing.assert_close(out, torch.tensor(want, dtype=torch.float64), rtol=1e-15, atol=1e-15)
    c2 = MFConv(1, 1, max_degree=4).double()
    grads = torch.autograd.grad(c2(x, ei).sum(), list(c2.parameters()))
    names = [n for n, _ in c2.named_parameters()]
    for n, g in zip(names, grads):
        assert g is not None
        if n.split(".")[1] in ("2", "4"):                    # degrees 0, 1 and 3 occur
            assert not g.any(), n


def _golden(golden_dir, kind):
    return torch.load(golden_dir + "/models_%s.pt" % kind)


def _check(m, c):
    check_golden_case(m, c, lambda: golden_data(c["inputs"]), pred=(1e-6, 1e-5), loss=(1e-6, 0), grads=grad_close(1e-4, 1e-6))


def _oracle(cls, c):
    case = dict(c, cfg={k: v for k, v in c["cfg"].items() if k != "initial_bias"})
    return oracle_from_case(cls, case)


@pytest.mark.parametrize("name", SAGE_CASES)
def test_sage_oracle_stack_matches_reference_golden(golden_dir, name):
    _check(_oracle(SAGEStackOracle, _golden(golden_dir, "sage")[name]), _golden(golden_dir, "sage")[name])


@pytest.mark.parametrize("name", MFC_CASES)
def test_mfc_oracle_stack_matches_reference_golden(golden_dir, name):
    c = _golden(golden_dir, "mfc")[name]
    _check(_oracle(MFCStackOracle, c), c)


def test_golden_graphs_cover_the_degree_corner_cases(golden_dir):
    """Isolated nodes, self-loops, duplicate edges and a node whose in-degree exceeds max_degree are in every case's graph."""
    for kind in ("sage", "mfc"):
        for name, c in _golden(golden_dir, kind).items():
            ei = c["inputs"]["edge_index"]
            n = c["inputs"]["x"].shape[0]
            deg = torch.bincount(ei[1], minlength=n)
            assert (deg == 0).any() and (ei[0] == ei[1]).any() and int(deg.max()) > 5, name
            assert torch.unique(ei, dim=1).shape[1] < ei.shape[1], name
