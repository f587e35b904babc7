"""EXECUTED drop-in (VERDICT r1 "missing" #3): the reference's OWN ``create_model_config`` / ``create_model``
(hydragnn/models/create.py:41-108,112-766) with the three-line dispatch of INTEGRATION.md inserted returns the engine's model, and
that model is interchangeable with the one the reference builds itself.  tests/golden/make_dropin_golden.py ran the reference's
code (AST-extracted, never copied; absent third-party packages stubbed as make_golden.py does) with ``HYDRAGNN_ENGINE`` unset and
set, and stored the keyword arguments the dispatch hands to ``hydragnn_b200.create_model`` together with what the reference's own
model shows the training loop.  CPU test -- constructing models and reading the plugin surface needs no CUDA.

Both checkpoint directions are covered without the reference at test time: the reference's checkpoint loads strictly into the
engine model, and the engine's state dict has exactly the reference's parameter names and shapes, which is what a strict
``load_state_dict`` into the reference model checks.  An unknown ``mpnn_type`` is not taken by the dispatch and falls through to
the reference's own code, whose ``ValueError`` the generator recorded.

Checked: same parameter names, shapes AND values (both sides seed with ``torch.manual_seed(0)``, create.py:164), and every attribute the
reference's train / validate / test loop reads through ``model.module`` (train_validate_test.py:225-242,498,731,736,1006-1018).
The PNA, PNAPlus, CGCNN and GAT configurations of tests/golden/make_{pna,pnaplus,cgcnn,gat}_golden.py are checked the same way,
with their BatchNorm feature layers (stack_support.check_dropin).
"""
import os
import sys

import pytest
import torch

from hydragnn_b200.cgcnn import CGCNNStack
from hydragnn_b200.gat import GATStack
from hydragnn_b200.pna import PNAStack
from hydragnn_b200.pnaplus import PNAPlusStack
from stack_support import check_dropin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _config(mpnn_type, mlip):
    """config["NeuralNetwork"] after update_config, LennardJones-like (examples/LennardJones/LJ.json with mpnn_type switched)"""
    arch = dict(mpnn_type=mpnn_type, input_dim=1, hidden_dim=32, output_dim=[1], pe_dim=0, global_attn_engine=None, global_attn_type=None,
                global_attn_heads=0, output_type=["node"] if mlip else ["graph"], activation_function="relu", task_weights=[1.0],
                num_conv_layers=2, freeze_conv_layers=False, initial_bias=None, num_nodes=None, max_neighbours=5, edge_dim=None,
                pna_deg=None, num_before_skip=None, num_after_skip=None, num_radial=5, radial_type=None, distance_transform=None,
                basis_emb_size=None, int_emb_size=None, out_emb_size=None, envelope_exponent=None, num_spherical=None,
                num_gaussians=None, num_filters=None, radius=5.0, equivariance=False, correlation=None, max_ell=None, node_max_ell=None,
                avg_num_neighbors=None)
    if mlip:
        # heads in the list-of-branches form that update_config produces (hydragnn/utils/model/model.py:314-349)
        arch.update(output_heads={"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [60, 20],
                                                                                  "type": "mlp"}}]},
                    enable_interatomic_potential=True, energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
    else:
        arch.update(output_heads={"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5,
                                                                                   "num_headlayers": 2, "dim_headlayers": [50, 25]}}]})
    return {"Architecture": arch, "Training": {"loss_function_type": "mse", "conv_checkpointing": False, "precision": "fp32"}}


@pytest.mark.parametrize("mpnn_type,mlip", [("EGNN", True), ("PAINN", False), ("EGNN", False)])
def test_reference_create_model_config_dispatches_to_the_engine(golden_dir, mpnn_type, mlip):
    sys.path.insert(0, ROOT)
    import hydragnn_b200 as hb
    g = torch.load(os.path.join(golden_dir, "dropin.pt"))["%s-%s" % (mpnn_type, mlip)]
    assert g["kwargs"]["mpnn_type"] == mpnn_type and mpnn_type in hb.create.SUPPORTED   # the dispatch takes this config
    eng = hb.create_model(**g["kwargs"])                                             # what the dispatch returns
    inner = eng.model if mlip else eng
    assert type(inner).__module__.startswith("hydragnn_b200"), type(inner)
    # same plugin surface as the reference's own model: parameter names, shapes and seeded values
    sr, se = g["state_dict"], eng.state_dict()
    assert list(sr.keys()) == list(se.keys())
    for k in sr:
        assert sr[k].shape == se[k].shape and torch.equal(sr[k], se[k]), k
    # what train() / validate() / test() read through model.module
    for attr, want in g["attrs"].items():
        assert hasattr(eng, attr), attr
        assert getattr(eng, attr) == want, attr
    assert hasattr(eng, "loss")
    if mlip:
        for attr in ("energy_force_loss", "energy_weight", "energy_peratom_weight", "force_weight"):
            assert hasattr(eng, attr), attr
        assert (eng.energy_weight, eng.energy_peratom_weight, eng.force_weight) == tuple(g["mlip_weights"]) == (1.0, 1.0, 1.0)
    # unknown mpnn_type: the dispatch leaves it to the reference, which raises its own error (create.py:584)
    assert "NOPE" not in hb.create.SUPPORTED and g["unknown_mpnn_type_error"] == "ValueError"
    # a reference checkpoint loads into the engine model (strict) and comes back out unchanged
    ref_inner = {k[len("model."):] if mlip else k: v for k, v in sr.items()}
    inner.load_state_dict(ref_inner, strict=True)
    assert all(torch.equal(v, ref_inner[k]) for k, v in inner.state_dict().items())
    # and the other direction: a strict load into the reference model needs exactly its names and shapes
    assert {k: tuple(v.shape) for k, v in inner.state_dict().items()} == {k: tuple(v.shape) for k, v in ref_inner.items()}
    assert str(inner) == g["repr"]


# (golden file, configuration, engine stack, its str): the reference's PNAStack and PNAPlusStack both print "PNAStack"
STACK_DROPIN = [("dropin_pna.pt", "PNA-edge1-node", PNAStack, "PNAStack"), ("dropin_pna.pt", "PNA-noedge-graph", PNAStack, "PNAStack"),
                ("dropin_pnaplus.pt", "PNAPlus-edge1-node", PNAPlusStack, "PNAStack"),
                ("dropin_pnaplus.pt", "PNAPlus-noedge-graph", PNAPlusStack, "PNAStack"),
                ("dropin_cgcnn.pt", "CGCNN-edge1-node", CGCNNStack, "CGCNNStack"),
                ("dropin_cgcnn.pt", "CGCNN-edge0-graph", CGCNNStack, "CGCNNStack"),
                ("dropin_cgcnn.pt", "CGCNN-gps-edge0-graph", CGCNNStack, "CGCNNStack"),
                ("dropin_gat.pt", "GAT-edge1-node", GATStack, "GATStack"), ("dropin_gat.pt", "GAT-noedge-graph", GATStack, "GATStack"),
                ("dropin_gat.pt", "GAT-gps-noedge-graph", GATStack, "GATStack")]


@pytest.mark.parametrize("golden,key,cls,name", STACK_DROPIN, ids=[k for _, k, _, _ in STACK_DROPIN])
def test_reference_create_model_config_dispatches_the_stack_to_the_engine(golden_dir, golden, key, cls, name):
    """PNA (EAM-like: 1-wide edge attribute, node head; no edge attributes, graph head), PNAPlus (the same), CGCNN (after
    update_config: hidden_dim = input_dim = 1 without GPS, edge_dim 0 or 1; GPS with edge_dim 0) and GAT (edge_dim None without
    edge features, 1 with the edge length; GPS without edge features): the engine's model is interchangeable with the reference's
    own stack, whose PyG conv is restated in oracle/."""
    check_dropin(torch.load(os.path.join(golden_dir, golden))[key], cls, name)
