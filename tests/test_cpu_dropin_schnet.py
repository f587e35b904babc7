"""The reference's own ``create_model_config`` with the INTEGRATION.md dispatch returns the engine's SCFStack for SchNet
configurations (qm9-like with GPS; equivariant MLIP with a node head), and that model is interchangeable with the reference's
own: same state-dict names, shapes and seeded values, same plugin attributes and ``str``, and a reference checkpoint loads into
it strictly.  tests/golden/make_schnet_golden.py wrote dropin_schnet.pt by running the reference's code.  CPU test."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200.schnet import SCFStack
from stack_support import check_dropin

KEYS = ["SchNet-gps-graph", "SchNet-equivariant-mlip"]


def _golden(golden_dir, key):
    return torch.load(golden_dir + "/dropin_schnet.pt")[key]


@pytest.mark.parametrize("key", KEYS)
def test_reference_create_model_config_dispatches_schnet_to_the_engine(golden_dir, key):
    eng = check_dropin(_golden(golden_dir, key), SCFStack, "SCFStack", batch_norm=False)
    assert "distance_expansion.offset" in getattr(eng, "model", eng).state_dict()


def test_in_layer_and_edge_index_branches_are_named_like_the_reference(golden_dir):
    eq = hb.create_model(**_golden(golden_dir, "SchNet-equivariant-mlip")["kwargs"]).model
    assert not eq.use_edge_attr and not eq.use_global_attn
    keys = eq.state_dict().keys()
    assert "graph_convs.0.module_1.offset" in keys and "graph_convs.0.module_2.lin1.weight" in keys
    assert "graph_convs.0.module_2.coord_mlp.2.weight" in keys and not any(k.startswith("graph_convs.1.module_2.coord") for k in keys)
    gps = hb.create_model(**_golden(golden_dir, "SchNet-gps-graph")["kwargs"])
    assert "graph_convs.0.conv.module_0.nn.0.weight" in gps.state_dict()


@pytest.mark.parametrize("missing,message", [("num_gaussians", "SchNet requires num_guassians input."),
                                             ("num_filters", "SchNet requires num_filters input."),
                                             ("radius", "SchNet requires radius input.")])
def test_schnet_requires_its_three_arguments(golden_dir, missing, message):
    kw = dict(_golden(golden_dir, "SchNet-gps-graph")["kwargs"], **{missing: None})
    with pytest.raises(AssertionError, match=message):
        hb.create_model(**kw)


def test_padded_step_refuses_schnet(golden_dir):
    from hydragnn_b200 import padded
    for key in KEYS:
        assert not padded.supported(hb.create_model(**_golden(golden_dir, key)["kwargs"]))
    # the non-GPS edge_dim > 0 branch reads data.edge_index; it is refused as well and runs eagerly
    kw = dict(_golden(golden_dir, "SchNet-equivariant-mlip")["kwargs"], edge_dim=1, equivariance=False)
    assert not padded.supported(hb.create_model(**kw))


def test_max_neighbours_none_is_refused_on_the_in_layer_branch(golden_dir):
    from hydragnn_b200.data import Batch, Data
    m = hb.create_model(**dict(_golden(golden_dir, "SchNet-equivariant-mlip")["kwargs"], max_neighbours=None)).model
    b = Batch.from_data_list([Data(x=torch.ones(3, 1), pos=torch.rand(3, 3))])
    with pytest.raises(ValueError, match="max_neighbours"):
        m._embedding(b, None, False)


def test_examples_configs_build_the_engine_stack():
    """examples/qm9/qm9.json and examples/md17/md17.json with input_dim / output_dim filled in as update_config does."""
    for layers, pe in ((2, 2), (6, 6)):
        arch = dict(mpnn_type="SchNet", input_dim=1, hidden_dim=64, output_dim=[1], pe_dim=pe, global_attn_engine="GPS",
                    global_attn_type="multihead", global_attn_heads=8, output_type=["graph"], activation_function="relu",
                    task_weights=[1.0], num_conv_layers=layers, max_neighbours=5, radius=7.0, num_gaussians=10, num_filters=8,
                    output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 10, "num_headlayers": 2,
                                            "dim_headlayers": [10, 10]}})
        m = hb.create_model_config({"Architecture": arch, "Training": {"loss_function_type": "mse"}}, use_gpu=False)
        assert isinstance(m, SCFStack) and len(m.graph_convs) == layers
