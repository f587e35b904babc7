"""Branch-weighted prediction of multi-branch interatomic potentials, host side (no GPU).

* oracle/branch_mix.py against the reference's own per-branch forward, ``_weighted_average`` and ``_fused_energy_forces``
  (tests/golden/models_branch_mix.pt, tests/golden/make_branch_mix_golden.py); the per-branch and fused forms agree in fp64.
* The all-branch ``BranchGroups`` layout: every row in every branch's group.
* Every refusal of ``branch_weighted_energy_forces`` / ``PaddedPredictStep`` and of the all-branch decoding.
"""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import stacks
from hydragnn_b200.data import Batch
from oracle import branch_mix as obm
from oracle.base import oracle_from_case
from stack_support import golden_data

CASES = ["egnn_graph", "egnn_node", "painn_graph", "painn_node"]
GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 7]}
NODE = {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}
MLIP = dict(enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden(golden_dir, name):
    c = torch.load(golden_dir + "/models_branch_mix.pt")[name]
    m = oracle_from_case(c["cfg"]["mpnn_type"], c).eval()
    d = golden_data(c["inputs"])
    d.pos.requires_grad_(True)
    w = c["weights"].double()
    energies, forces = obm.per_branch(m, d, 3)
    torch.testing.assert_close(energies.T, c["branch_energy"].double(), rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(forces, c["branch_forces"].double(), rtol=1e-4, atol=1e-8)
    e_avg, f_avg = obm.weighted_average(energies, forces, w, d.batch)
    torch.testing.assert_close(e_avg, c["avg_energy"].double(), rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(f_avg, c["avg_forces"].double(), rtol=1e-4, atol=1e-8)
    e_fused, f_fused = obm.fused(m, d, w)
    torch.testing.assert_close(e_fused, c["fused_energy"].double(), rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(f_fused, c["fused_forces"].double(), rtol=1e-4, atol=1e-8)
    # one backward of the weighted energy = the weighted average of the per-branch forces, in fp64
    torch.testing.assert_close(e_fused, e_avg, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(f_fused, f_avg, rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("rows,branches", [(4, 3), (1, 1), (0, 2), (5, 17)])
def test_all_branch_groups_layout(rows, branches):
    g = stacks.all_branch_groups(rows, branches, "cpu")
    assert g.rowptr.tolist() == [b * rows for b in range(branches + 1)]
    j = torch.arange(rows * branches)
    assert torch.equal(g.order.idx.long(), j % max(rows, 1))                # sorted row b R + r is row r ...
    assert torch.equal(g.rows.idx.long(), j // max(rows, 1))                # ... in branch b
    assert g.order.n == rows and g.rows.n == branches
    # the adjoint of the replication sums every row's copies: the CSR by row lists its copies in branch order
    assert g.order.rowptr.tolist() == [r * branches for r in range(rows + 1)]
    for r in range(rows):
        copies = g.order.perm[g.order.rowptr[r]:g.order.rowptr[r + 1]].tolist()
        assert copies == [b * rows + r for b in range(branches)]


def _model(kinds=("graph",), graph=None, node=None, mlip=True, pooling=None, **kw):
    heads = {"graph": graph or [{"type": "branch-%d" % b, "architecture": dict(GRAPH)} for b in range(3)]}
    if node is not None:
        heads["node"] = node
    base = dict(mpnn_type="EGNN", input_dim=1, hidden_dim=8, num_conv_layers=2, num_radial=5, radius=5.0)
    base.update(kw)
    m = hb.create_model(**base, output_dim=[1] * len(kinds), output_type=list(kinds), task_weights=[1.0] * len(kinds),
                        output_heads=heads, graph_pooling=pooling or ("add" if kinds[0] == "graph" else "mean"), use_gpu=False,
                        **(MLIP if mlip else {}))
    return m.eval()


def _data(g=2):
    d = Batch(x=torch.ones(3 * g, 1), pos=torch.zeros(3 * g, 3), batch=torch.arange(g).repeat_interleave(3),
              edge_index=torch.zeros(2, 0, dtype=torch.int64))
    d._num_graphs = g
    return d


def _refused(model, weights, match, data=None):
    with pytest.raises(ValueError, match=match):
        hb.branch_weighted_energy_forces(model, data if data is not None else _data(), weights)


def test_refusals():
    w = torch.full((2, 3), 1 / 3)
    _refused(_model().train(), w, "eval mode")
    _refused(_model(mlip=False), w, "interatomic potential")
    m = _model()
    m.model.var_output = 1
    _refused(m, w, "mean-and-variance")
    _refused(_model(pooling="mean"), w, "sum pooling")
    differ = [{"type": "branch-%d" % b, "architecture": dict(GRAPH)} for b in range(3)]
    differ[1]["architecture"]["dim_headlayers"] = [10, 8]
    _refused(_model(graph=differ), w, "share one architecture")
    node_differ = [{"type": "branch-%d" % b, "architecture": dict(NODE)} for b in range(3)]
    node_differ[2]["architecture"]["dim_headlayers"] = [12, 5]
    _refused(_model(kinds=("node",), node=node_differ), w, "share one architecture")
    m = _model()
    _refused(m, torch.full((2, 2), 0.5), "float32 \\[graphs, branches\\] = \\[2, 3\\]")          # branches
    _refused(m, torch.full((3, 3), 0.5), "= \\[2, 3\\]")                                           # graphs
    _refused(m, w.double(), "float32")
    _refused(m, w.to("meta"), "on cpu")
    _refused(m, [[1.0] * 3] * 2, "list")
    _refused(m, w.clone().requires_grad_(True), "must not require grad")
    with pytest.raises(ValueError, match="eval mode"):
        hb.PaddedPredictStep(_model().train(), _data())
    with pytest.raises(ValueError, match="share one architecture"):
        hb.PaddedPredictStep(_model(graph=differ), _data())


def test_all_branch_decoding_refuses_branches_that_differ():
    """Under ``all_branches()`` a head whose branches differ raises instead of falling back to per-branch masks."""
    differ = [{"type": "branch-%d" % b, "architecture": dict(GRAPH)} for b in range(3)]
    differ[1]["architecture"]["dim_headlayers"] = [10, 8]
    inner = _model(graph=differ).model
    plan = stacks.AllBranchPlan(2, 6, 3, "cpu")
    with pytest.raises(ValueError, match="share one architecture"):
        stacks.grouped_decode("graph", inner.heads_NN[0], inner.graph_shared, plan, torch.zeros(6, 8), torch.zeros(2, 8), 1, False)
