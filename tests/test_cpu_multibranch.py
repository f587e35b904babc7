"""Multi-branch heads on the captured padded step, host side (no GPU): which models ``padded.supported`` accepts, and how
``dataset_name`` travels in a padded batch."""
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import padded
from hydragnn_b200.data import Batch

GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 7]}
NODE = {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}
MLIP = dict(enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
MACE = dict(mpnn_type="MACE", input_dim=1, hidden_dim=8, num_conv_layers=2, num_radial=8, radius=6.0, max_ell=2, node_max_ell=1,
            avg_num_neighbors=10.0, envelope_exponent=5, correlation=2, num_nodes=9)


def branches(arch, n=3, differ=None):
    out = [{"type": "branch-%d" % b, "architecture": dict(arch)} for b in range(n)]
    if differ is not None:
        out[1]["architecture"]["dim_headlayers"] = differ
    return out


def model(mpnn_type="EGNN", kinds=("graph",), graph=None, node=None, mlip=False, **kw):
    heads = {}
    if graph is not None:
        heads["graph"] = graph
    if node is not None:
        heads["node"] = node
    base = dict(mpnn_type=mpnn_type, input_dim=1, hidden_dim=8, num_conv_layers=2, num_radial=5, radius=5.0)
    base.update(kw)
    return hb.create_model(**base, output_dim=[1] * len(kinds), output_type=list(kinds), task_weights=[1.0] * len(kinds),
                           output_heads=heads, graph_pooling="add" if mlip and kinds[0] == "graph" else "mean",
                           use_gpu=False, **(MLIP if mlip else {}))


def test_supported_accepts_branches_that_share_one_architecture():
    assert padded.supported(model(graph=branches(GRAPH, 1)))                               # one branch: as before
    assert padded.supported(model(graph=branches(GRAPH)))                                  # graph heads, 3 branches
    assert padded.supported(model("PAINN", graph=branches(GRAPH)))
    assert padded.supported(model(kinds=("graph",), graph=branches(GRAPH), mlip=True))      # MLIP, graph energy head
    assert padded.supported(model(kinds=("node",), graph=branches(GRAPH), node=branches(NODE), mlip=True))
    assert padded.supported(model(**MACE, kinds=("node",), graph=branches(GRAPH), node=branches(NODE), mlip=True))
    assert padded.supported(model(**MACE, kinds=("graph",), graph=branches(GRAPH), node=branches(NODE), mlip=True))


def test_supported_refuses_branches_that_differ():
    assert not padded.supported(model(graph=branches(GRAPH, differ=[10, 8])))
    assert not padded.supported(model(kinds=("graph",), graph=branches(GRAPH, differ=[9, 7]), mlip=True))
    assert not padded.supported(model(kinds=("node",), graph=branches(GRAPH), node=branches(NODE, differ=[12, 5]), mlip=True))
    assert not padded.supported(model(**MACE, kinds=("node",), graph=branches(GRAPH), node=branches(NODE, differ=[12, 5]),
                                      mlip=True))
    # node heads outside the MLIP wrapper stay eager, with one branch or several
    assert not padded.supported(model(kinds=("graph", "node"), graph=branches(GRAPH, 1), node=branches(NODE, 1)))
    assert not padded.supported(model(kinds=("graph", "node"), graph=branches(GRAPH), node=branches(NODE)))


def _batch(g, with_names=True):
    b = Batch(x=torch.ones(3 * g, 1), pos=torch.zeros(3 * g, 3), batch=torch.arange(g).repeat_interleave(3),
              edge_index=torch.zeros(2, 0, dtype=torch.int64), y=torch.zeros(g, 1))
    b._num_graphs = g
    if with_names:
        b.dataset_name = torch.tensor([[2], [0], [1], [2]])[:g]
    return b


def test_dataset_name_is_a_graph_field_of_multi_branch_models_only():
    multi, single = model(graph=branches(GRAPH)), model(graph=branches(GRAPH, 1))
    fields = padded.batch_fields(multi, _batch(4), False)
    assert fields["dataset_name"] == ((1,), torch.int64)
    assert "dataset_name" not in padded.batch_fields(single, _batch(4), False)       # one branch: the batch carries what it did
    try:
        padded.batch_fields(multi, _batch(4, with_names=False), False)
    except ValueError as e:
        assert "dataset_name" in str(e)
    else:
        raise AssertionError("a multi-branch model needs dataset_name")


def test_filler_graphs_decode_with_branch_zero():
    buf = torch.full((7, 1), 5, dtype=torch.int64)              # what the previous batch left in the staging buffer
    padded.stage(buf, "dataset_name", torch.tensor([[2], [0], [1]], dtype=torch.int32), 3, 9, 10)
    assert buf.dtype == torch.int64 and buf.reshape(-1).tolist() == [2, 0, 1, 0, 0, 0, 0]
    flat = torch.full((5, 1), 5, dtype=torch.int64)
    padded.stage(flat, "dataset_name", torch.tensor([1, 2]), 2, 6, 8)                   # a 1-D dataset_name becomes one column
    assert flat.reshape(-1).tolist() == [1, 2, 0, 0, 0]
