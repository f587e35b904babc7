"""SAGE and MFC through the engine's construction on the CPU: the reference's own ``create_model_config`` with the INTEGRATION.md
dispatch returns the engine's SAGEStack / MFCStack, with the reference's state-dict names, shapes and seeded values, plugin
attributes and ``str``; checkpoints load strictly both ways; the reference's refusals are the engine's.  tests/golden/
make_sage_mfc_golden.py wrote the goldens by running the reference's code; PyG's convs are restated there (oracle/sage.py)."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import padded
from hydragnn_b200.sage import MFCStack, SAGEStack
from oracle.base import case_kwargs, oracle_from_case
from stack_support import check_dropin, check_seeded_state

DROPIN = ["SAGE-graph-bias", "SAGE-node", "SAGE-gps-graph", "MFC-node-bias", "MFC-node", "MFC-gps-graph"]
STACKS = {"SAGE": SAGEStack, "MFC": MFCStack}


def _dropin(golden_dir):
    return torch.load(golden_dir + "/dropin_sage_mfc.pt")


@pytest.mark.parametrize("key", DROPIN)
def test_reference_create_model_config_dispatches_to_the_engine(golden_dir, key):
    kind = key.split("-")[0]
    assert not padded.supported(check_dropin(_dropin(golden_dir)[key], STACKS[kind], kind + "Stack"))


def _cases(golden_dir, kind):
    return torch.load(golden_dir + "/models_%s.pt" % kind.lower())


@pytest.mark.parametrize("kind", ["SAGE", "MFC"])
def test_engine_state_dicts_match_every_golden_case_and_load_both_ways(golden_dir, kind):
    """Seeded construction of every case equals the reference's (names, order, shapes, values; SAGE ignores initial_bias, MFC
    honours it), the reference's checkpoint loads strictly into the engine, and the engine's into the oracle stack."""
    for name, c in _cases(golden_dir, kind).items():
        eng = hb.create_model(**case_kwargs(kind, c), use_gpu=False)
        assert type(eng) is STACKS[kind] and str(eng) == c["str"], name
        check_seeded_state(eng, c["state"])
        oracle_from_case(kind, c, state=eng.state_dict())


def test_mfc_requires_max_neighbours(golden_dir):
    err = _dropin(golden_dir)["errors"]["mfc_no_max_neighbours"]
    assert err["type"] == "AssertionError" and err["msg"] == "MFC requires max_neighbours input."
    g = _dropin(golden_dir)["MFC-node"]["kwargs"]
    with pytest.raises(AssertionError, match="^MFC requires max_neighbours input.$"):
        hb.create_model(**dict(g, max_neighbours=None))


def test_initial_bias_sage_ignores_it_mfc_fills_the_graph_heads_like_every_engine_stack(golden_dir):
    """create.py does not pass initial_bias to SAGEStack.  MFC receives it; the reference's Base._set_bias then fails on the graph
    head's branch dict (recorded in the golden, as it fails for every stack), while the engine's Base fills the last bias of every
    graph branch, as it does for PNA, GAT and the rest."""
    d = _dropin(golden_dir)
    sage = hb.create_model(**d["SAGE-graph-bias"]["kwargs"])
    assert d["SAGE-graph-bias"]["kwargs"]["initial_bias"] == 0.5
    assert not any(torch.all(p == 0.5) for n, p in sage.state_dict().items() if n.startswith("heads_NN") and n.endswith("bias"))
    assert d["errors"]["mfc_initial_bias_graph"]["type"] == "KeyError"
    kw = dict(d["MFC-node"]["kwargs"], output_type=["graph"], output_heads=d["SAGE-graph-bias"]["kwargs"]["output_heads"],
              initial_bias=0.5)
    mfc = hb.create_model(**kw)
    pna = hb.create_model(**dict(kw, mpnn_type="PNA", pna_deg=[0, 1, 2]))
    for m in (mfc, pna):
        assert torch.all(m.heads_NN[0]["branch-0"][-1].bias == 0.5)


def test_gin_and_dimenet_are_still_unknown():
    g = dict(input_dim=1, hidden_dim=8, output_dim=[1], output_type=["graph"], use_gpu=False,
             output_heads={"graph": {"num_sharedlayers": 1, "dim_sharedlayers": 4, "num_headlayers": 1, "dim_headlayers": [4]}})
    for t in ("GIN", "DimeNet"):
        with pytest.raises(ValueError, match="Unknown mpnn_type"):
            hb.create_model(mpnn_type=t, **g)
