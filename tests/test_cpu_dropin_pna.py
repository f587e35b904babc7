"""The engine's PNA construction on the CPU against dropin_pna.pt (tests/golden/make_pna_golden.py ran the reference's own
``create_model_config``; the dispatch itself is checked in tests/test_cpu_dropin.py): the reference's refusals.  CPU test."""
import pytest
import torch

import hydragnn_b200 as hb


def test_pna_requires_degree_input(golden_dir):
    g = torch.load(golden_dir + "/dropin_pna.pt")["PNA-noedge-graph"]
    with pytest.raises(AssertionError, match="PNA requires degree input"):
        hb.create_model(**dict(g["kwargs"], pna_deg=None))


def test_padded_step_refuses_batchnorm_feature_layers(golden_dir):
    from hydragnn_b200 import padded
    g = torch.load(golden_dir + "/dropin_pna.pt")["PNA-noedge-graph"]
    assert not padded.supported(hb.create_model(**g["kwargs"]))
