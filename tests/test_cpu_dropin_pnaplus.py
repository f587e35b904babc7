"""The engine's PNAPlus construction on the CPU against dropin_pnaplus.pt (tests/golden/make_pnaplus_golden.py ran the reference's
own ``create_model_config``; the dispatch itself is checked in tests/test_cpu_dropin.py): ``rbf.freq`` last in the state dict,
``envelope_exponent`` forwarded by the engine's ``create_model_config``, and the reference's refusals.  CPU test."""
import pytest
import torch

import hydragnn_b200 as hb


@pytest.mark.parametrize("key", ["PNAPlus-edge1-node", "PNAPlus-noedge-graph"])
def test_rbf_freq_is_the_last_state_dict_entry(golden_dir, key):
    g = torch.load(golden_dir + "/dropin_pnaplus.pt")[key]
    assert list(g["state_dict"].keys())[-1] == "rbf.freq" == list(hb.create_model(**g["kwargs"]).state_dict().keys())[-1]


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
