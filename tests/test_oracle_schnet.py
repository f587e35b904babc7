"""oracle/schnet.py pinned by hand-computed cases, and its CFConv checked against the reference's own stack
(models_schnet.pt, written by tests/golden/make_schnet_golden.py).  CPU test."""
import math

import torch

import pytest

from oracle import schnet as so
from oracle.base import oracle_from_case
from stack_support import check_golden_case, golden_data, grad_norm


def test_gaussian_coefficient_and_values():
    g = so.GaussianSmearing(0.0, 7.0, 10)
    step = 7.0 / 9.0
    assert abs(g.coeff - (-0.5 / ((torch.tensor(7.0) / 9).item() ** 2))) < 1e-12
    assert abs(g.coeff + 0.5 / step ** 2) < 1e-5
    v = g(torch.tensor([step]))
    assert abs(float(v[0, 1]) - 1.0) < 1e-6 and abs(float(v[0, 0]) - math.exp(-0.5)) < 1e-6


def test_shifted_softplus_on_both_sides_of_the_threshold():
    s = so.ShiftedSoftplus()
    x = torch.tensor([0.0, 1.0, 19.5, 20.5, -30.0], dtype=torch.float64)
    y = s(x)
    ln2 = torch.log(torch.tensor(2.0)).item()
    assert abs(float(y[0])) < 1e-7
    assert abs(float(y[1]) - (math.log1p(math.exp(1.0)) - ln2)) < 1e-12
    assert abs(float(y[2]) - (math.log1p(math.exp(19.5)) - ln2)) < 1e-12
    assert float(y[3]) == 20.5 - ln2                       # above the threshold softplus is the identity
    assert abs(float(y[4]) + ln2) < 1e-12


def test_envelope_past_the_cutoff_is_not_zero():
    pos = torch.tensor([[0.0, 0.0, 0.0], [1.5, 0.0, 0.0]], dtype=torch.float64)
    ei = torch.tensor([[0], [1]])
    nf, g = 2, 3
    w1 = torch.zeros(nf, g, dtype=torch.float64)
    b1 = torch.zeros(nf, dtype=torch.float64)
    w2 = torch.zeros(nf, nf, dtype=torch.float64)
    b2 = torch.ones(nf, dtype=torch.float64)
    eye = torch.eye(nf, dtype=torch.float64)
    x = torch.tensor([[1.0, 2.0], [0.0, 0.0]], dtype=torch.float64)
    out, w = so.cfconv(x, pos, ei, eye, w1, b1, w2, b2, eye, torch.zeros(nf, dtype=torch.float64),
                       torch.linspace(0, 1, g, dtype=torch.float64), -2.0, 1.0)
    c = 0.5 * (math.cos(1.5 * math.pi) + 1.0)             # d = 1.5 > cutoff 1: 0.5, not masked
    assert abs(c - 0.5) < 1e-12
    assert torch.allclose(w, torch.full((1, nf), c, dtype=torch.float64))
    assert torch.allclose(out[1], torch.tensor([1.0, 2.0], dtype=torch.float64) * c) and torch.all(out[0] == 0)


def test_coordinate_update_is_a_mean_over_sources():
    pos = torch.tensor([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.0, 3.0, 0.0]], dtype=torch.float64)
    ei = torch.tensor([[0, 0, 1], [1, 2, 2]])              # node 0 is the source of two edges, node 1 of one, node 2 of none
    w = torch.zeros(3, 1, dtype=torch.float64)
    new = so.coord_update(pos, ei, w, lambda t: torch.ones(t.shape[0], 1, dtype=t.dtype))
    d01, d02, d12 = torch.tensor([2.0, 0, 0]) / 3.0, torch.tensor([0, 3.0, 0]) / 4.0, torch.tensor([-2.0, 3.0, 0]) / (13 ** 0.5 + 1)
    assert torch.allclose(new[0], pos[0] + (d01 + d02).double() / 2)
    assert torch.allclose(new[1], pos[1] + d12.double())
    assert torch.equal(new[2], pos[2])


@pytest.mark.parametrize("name", ["inlayer_graph", "inlayer_truncated", "equivariant_conv_head", "edge_len", "edge3", "gps",
                                  "gps_edge2", "add_pool"])
def test_oracle_stack_matches_the_reference(golden_dir, name):
    """The oracle stack at fp64 against the reference's own SCFStack (fp32): eval predictions, the train-mode loss and every
    parameter gradient."""
    case = torch.load(golden_dir + "/models_schnet.pt")[name]
    # norm-wise gradients: a bias followed by BatchNorm has a zero true gradient, the reference's fp32 value there is rounding noise
    check_golden_case(oracle_from_case("SchNet", case), case, lambda: golden_data(case["inputs"]), pred=(1e-5, 1e-5),
                      loss=(1e-5, 0), grads=grad_norm(1e-4, 1e-6))
