"""The reference's own ``create_model_config`` with the INTEGRATION.md dispatch returns the engine's GAT model for GAT
configurations that went through update_config (edge_dim None without edge features, 1 with the edge length; and GPS without
edge features), and that model is interchangeable with the reference's own GATStack: same state-dict names, shapes and seeded values, same
plugin attributes and ``str``, and a reference checkpoint loads into it strictly.  tests/golden/make_gat_golden.py wrote
dropin_gat.pt by running the reference's code; PyG's GATv2Conv is restated there (oracle/gat.py).  CPU test."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200.gat import GATStack


@pytest.mark.parametrize("key", ["GAT-edge1-node", "GAT-noedge-graph", "GAT-gps-noedge-graph"])
def test_reference_create_model_config_dispatches_gat_to_the_engine(golden_dir, key):
    g = torch.load(golden_dir + "/dropin_gat.pt")[key]
    assert g["kwargs"]["mpnn_type"] == "GAT" and "GAT" in hb.create.SUPPORTED
    eng = hb.create_model(**g["kwargs"])
    assert isinstance(eng, GATStack)
    sr, se = g["state_dict"], eng.state_dict()
    assert list(sr.keys()) == list(se.keys())
    for k in sr:
        assert sr[k].shape == se[k].shape and torch.equal(sr[k], se[k]), k
    for attr, want in g["attrs"].items():
        assert getattr(eng, attr) == want, attr
    eng.load_state_dict(sr, strict=True)
    assert all(torch.equal(v, sr[k]) for k, v in eng.state_dict().items())
    assert str(eng) == g["repr"] == "GATStack"
    assert len(eng.feature_layers) == len(eng.graph_convs) == g["config"]["Architecture"]["num_conv_layers"]
