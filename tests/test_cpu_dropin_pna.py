"""The reference's own ``create_model_config`` with the INTEGRATION.md dispatch returns the engine's PNA model for PNA
configurations (EAM-like: 1-wide edge attribute, node head; and without edge attributes, graph head), and that model is
interchangeable with the reference's own PNAStack: same state-dict names, shapes and seeded values, same plugin attributes and
``str``, and a reference checkpoint loads into it strictly.  tests/golden/make_pna_golden.py wrote dropin_pna.pt by running the
reference's code; PyG's PNAConv is restated there (oracle/pna.py).  CPU test."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200.pna import PNAStack


@pytest.mark.parametrize("key", ["PNA-edge1-node", "PNA-noedge-graph"])
def test_reference_create_model_config_dispatches_pna_to_the_engine(golden_dir, key):
    g = torch.load(golden_dir + "/dropin_pna.pt")[key]
    assert g["kwargs"]["mpnn_type"] == "PNA" and "PNA" in hb.create.SUPPORTED
    eng = hb.create_model(**g["kwargs"])
    assert isinstance(eng, PNAStack)
    sr, se = g["state_dict"], eng.state_dict()
    assert list(sr.keys()) == list(se.keys())
    for k in sr:
        assert sr[k].shape == se[k].shape and torch.equal(sr[k], se[k]), k
    for attr, want in g["attrs"].items():
        assert getattr(eng, attr) == want, attr
    eng.load_state_dict(sr, strict=True)
    assert all(torch.equal(v, sr[k]) for k, v in eng.state_dict().items())
    assert str(eng) == g["repr"] == "PNAStack"
    # BatchNorm feature layers, one per conv, named like PyG's BatchNorm wrapper
    assert all(isinstance(f.module, torch.nn.BatchNorm1d) for f in eng.feature_layers)
    assert len(eng.feature_layers) == len(eng.graph_convs) == g["config"]["Architecture"]["num_conv_layers"]


def test_pna_requires_degree_input(golden_dir):
    g = torch.load(golden_dir + "/dropin_pna.pt")["PNA-noedge-graph"]
    with pytest.raises(AssertionError, match="PNA requires degree input"):
        hb.create_model(**dict(g["kwargs"], pna_deg=None))


def test_padded_step_refuses_batchnorm_feature_layers(golden_dir):
    from hydragnn_b200 import padded
    g = torch.load(golden_dir + "/dropin_pna.pt")["PNA-noedge-graph"]
    assert not padded.supported(hb.create_model(**g["kwargs"]))
