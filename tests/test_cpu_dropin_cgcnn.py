"""The reference's own ``create_model_config`` with the INTEGRATION.md dispatch returns the engine's CGCNN model for CGCNN
configurations that went through update_config (hidden_dim = input_dim = 1 without GPS, edge_dim 0 or 1; and GPS with edge_dim
0), and that model is interchangeable with the reference's own CGCNNStack: same state-dict names, shapes and seeded values, same
plugin attributes and ``str``, and a reference checkpoint loads into it strictly.  tests/golden/make_cgcnn_golden.py wrote
dropin_cgcnn.pt by running the reference's code; PyG's CGConv is restated there (oracle/cgcnn.py).  CPU test."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200.cgcnn import CGCNNStack


@pytest.mark.parametrize("key", ["CGCNN-edge1-node", "CGCNN-edge0-graph", "CGCNN-gps-edge0-graph"])
def test_reference_create_model_config_dispatches_cgcnn_to_the_engine(golden_dir, key):
    g = torch.load(golden_dir + "/dropin_cgcnn.pt")[key]
    assert g["kwargs"]["mpnn_type"] == "CGCNN" and "CGCNN" in hb.create.SUPPORTED
    eng = hb.create_model(**g["kwargs"])
    assert isinstance(eng, CGCNNStack)
    sr, se = g["state_dict"], eng.state_dict()
    assert list(sr.keys()) == list(se.keys())
    for k in sr:
        assert sr[k].shape == se[k].shape and torch.equal(sr[k], se[k]), k
    for attr, want in g["attrs"].items():
        assert getattr(eng, attr) == want, attr
    eng.load_state_dict(sr, strict=True)
    assert all(torch.equal(v, sr[k]) for k, v in eng.state_dict().items())
    assert str(eng) == g["repr"] == "CGCNNStack"
    assert len(eng.feature_layers) == len(eng.graph_convs) == g["config"]["Architecture"]["num_conv_layers"]
