"""The reference's own ``create_model_config`` with the INTEGRATION.md dispatch returns the engine's PNAPlus model for PNAPlus
configurations, interchangeable with the reference's PNAPlusStack: same state-dict names, shapes and seeded values (``rbf.freq``
last), plugin attributes and ``str``; a reference checkpoint loads strictly.  The engine's ``create_model_config`` forwards
``envelope_exponent``.  tests/golden/make_pnaplus_golden.py wrote dropin_pnaplus.pt by running the reference's code.  CPU test."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200.pnaplus import PNAPlusStack


@pytest.mark.parametrize("key", ["PNAPlus-edge1-node", "PNAPlus-noedge-graph"])
def test_reference_create_model_config_dispatches_pnaplus_to_the_engine(golden_dir, key):
    g = torch.load(golden_dir + "/dropin_pnaplus.pt")[key]
    assert g["kwargs"]["mpnn_type"] == "PNAPlus" and "PNAPlus" in hb.create.SUPPORTED
    eng = hb.create_model(**g["kwargs"])
    assert isinstance(eng, PNAPlusStack)
    sr, se = g["state_dict"], eng.state_dict()
    assert list(sr.keys()) == list(se.keys()) and list(se.keys())[-1] == "rbf.freq"
    for k in sr:
        assert sr[k].shape == se[k].shape and torch.equal(sr[k], se[k]), k
    for attr, want in g["attrs"].items():
        assert getattr(eng, attr) == want, attr
    eng.load_state_dict(sr, strict=True)
    assert str(eng) == g["repr"] == "PNAStack"
    assert all(isinstance(f.module, torch.nn.BatchNorm1d) for f in eng.feature_layers)


def test_create_model_config_forwards_envelope_exponent(golden_dir):
    g = torch.load(golden_dir + "/dropin_pnaplus.pt")["PNAPlus-noedge-graph"]
    assert g["config"]["Architecture"]["envelope_exponent"] == 3
    m = hb.create_model_config(g["config"], use_gpu=False)
    assert m.rbf.envelope.p == 4 and m.rbf.envelope_exponent == 3


@pytest.mark.parametrize("missing", ["pna_deg", "envelope_exponent", "num_radial", "radius"])
def test_pnaplus_requires_its_inputs(golden_dir, missing):
    g = torch.load(golden_dir + "/dropin_pnaplus.pt")["PNAPlus-noedge-graph"]
    with pytest.raises(AssertionError, match="PNAPlus requires"):
        hb.create_model(**dict(g["kwargs"], **{missing: None}))


def test_padded_step_refuses_pnaplus(golden_dir):
    from hydragnn_b200 import padded
    g = torch.load(golden_dir + "/dropin_pnaplus.pt")["PNAPlus-noedge-graph"]
    assert not padded.supported(hb.create_model(**g["kwargs"]))
