"""CPU tests of MACE graph-attribute conditioning: the fp64 restatement (oracle/mace.py) against
tests/golden/models_mace_cond.pt, which comes from the reference's own MACEStack (tests/golden/make_mace_cond_golden.py), and
the engine's lazily created modules, checkpoints and refusals -- all before any kernel runs."""
import pytest
import torch

import hydragnn_b200 as hb
from oracle.mace import MACEOracle
from stack_support import MACE_KW


def _golden(golden_dir):
    return torch.load(golden_dir + "/models_mace_cond.pt")


def _cases(golden_dir):
    """(name, case) with the shared parts of the file filled in: "state" (the whole state dict after the seeded first forward: the
    shared entries, then the conditioning modules') and "inputs" (the batch with the case's graph_attr)."""
    g = _golden(golden_dir)
    out = []
    for name, c in g["cases"].items():
        d = c["cfg"]["edge_dim"]
        base, cond = g["base_state"][d], c["cond_state"]
        out.append((name, dict(c, state={**base, **cond},
                               inputs=dict(g["batches"][d], graph_attr=c["graph_attr"]))))
    return out


def _batch(c):
    d = hb.Batch(**{k: v.clone() for k, v in c["inputs"].items()})
    d._num_graphs = 3
    return d


def _ga_dim(c):
    ga = c["graph_attr"]
    return ga.shape[1] if ga.dim() == 2 else ga.numel() // 3


def test_cond_oracle_matches_the_reference_own_code_golden(golden_dir):
    for name, c in _cases(golden_dir):
        torch.manual_seed(0)
        m = MACEOracle(**dict(MACE_KW, **c["cfg"]))
        m.eval()
        d = _batch(c)
        d.pos.requires_grad_(True)
        torch.manual_seed(1234)
        pred = m(d)
        sd = m.state_dict()
        assert list(sd.keys()) == list(c["state"].keys()), name
        for k, v in sd.items():
            assert torch.equal(v, c["state"][k]), (name, k)
        for p, q in zip(pred, c["pred"]):
            torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
        obj = pred[0].sum() + pred[1].pow(2).sum()
        f, = torch.autograd.grad(obj, d.pos, retain_graph=True)
        torch.testing.assert_close(f, c["dobj_dpos"], rtol=1e-4, atol=1e-7)
        grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            if n not in c["grads"]:          # recorded for a subset of the cases only (see make_mace_cond_golden.py)
                continue
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), (name, n)
            if gr is not None:
                torch.testing.assert_close(gr, ref, rtol=1e-4, atol=1e-6 * max(1.0, float(ref.abs().max())))


def _engine(cfg):
    return hb.create_model(mpnn_type="MACE", use_gpu=False, **dict(MACE_KW, **cfg))


def _ensure_as_load_existing_model(m, sd):
    """What hydragnn/utils/model/model.py:238-285 does before its strict load."""
    for key in sd:
        if key.endswith("graph_conditioner.0.weight") and m.graph_conditioner is None:
            m.use_graph_attr_conditioning = True
            m._ensure_graph_conditioner(sd[key].shape[1], m.device)
        if key.endswith("graph_concat_projector.weight") and m.graph_concat_projector is None:
            in_features = sd[key].shape[1]
            channel_dim = getattr(m, "hidden_dim", in_features)
            m.use_graph_attr_conditioning = True
            m.graph_attr_conditioning_mode = "concat_node"
            m._ensure_graph_concat_projector(graph_attr_dim=max(in_features - channel_dim, 1), channel_dim=channel_dim, device=m.device)


def test_engine_seeded_first_forward_state_matches_the_reference(golden_dir):
    """The engine draws the conditioning modules as the reference's first forward does: same names, order and values."""
    for name, c in _cases(golden_dir):
        m = _engine(c["cfg"])
        mode = c["cfg"]["graph_attr_conditioning_mode"]
        assert not m.graph_attr_modules_missing() or mode != "fuse_pool"
        torch.manual_seed(1234)
        if mode == "film":
            m._ensure_graph_conditioner(_ga_dim(c), m.device)
        elif mode == "concat_node":
            m._ensure_graph_concat_projector(graph_attr_dim=_ga_dim(c), channel_dim=m.hidden_dim, device=m.device)
        assert not m.graph_attr_modules_missing()
        se, params = m.state_dict(), dict(m.named_parameters())
        assert list(se.keys()) == list(c["state"].keys()), name
        for k, v in se.items():
            if k in params:
                assert torch.equal(v, c["state"][k]), (name, k)
            else:
                assert torch.allclose(v, c["state"][k], atol=1e-6), (name, k)


def test_conditioned_checkpoints_load_strictly_both_ways(golden_dir):
    for name, c in _cases(golden_dir):
        if c["cfg"]["graph_attr_conditioning_mode"] == "fuse_pool":
            continue
        fresh = _engine(c["cfg"])
        _ensure_as_load_existing_model(fresh, c["state"])
        fresh.load_state_dict(c["state"], strict=True)
        o = MACEOracle(**dict(MACE_KW, **c["cfg"]))
        _ensure_as_load_existing_model(o, fresh.state_dict())
        o.load_state_dict(fresh.state_dict(), strict=True)
        for k, v in o.state_dict().items():
            assert torch.equal(v, c["state"][k]), (name, k)


def test_every_refusal_matches_the_reference_before_any_kernel(golden_dir):
    ref = _golden(golden_dir)["refusals"]
    with pytest.raises(ValueError) as e:
        _engine(dict(use_graph_attr_conditioning=True, graph_attr_conditioning_mode="sum"))
    assert str(e.value) == ref["bad_mode"]["msg"]
    m = _engine(dict(use_graph_attr_conditioning=True, graph_attr_conditioning_mode="concat_node"))
    for key in ("missing", "1d_not_divisible", "2d_wrong_rows", "3d"):
        d = hb.Batch(graph_attr=ref[key]["graph_attr"])
        with pytest.raises(ValueError) as e:
            m._graph_attr(d, 3, torch.zeros(1))
        assert str(e.value) == ref[key]["msg"], key
    # and through forward: the check comes before the first kernel (this CPU model would fail at the first kernel otherwise)
    d = hb.Batch(x=torch.ones(4, 1), pos=torch.zeros(4, 3), edge_index=torch.zeros(2, 0, dtype=torch.long),
                 batch=torch.zeros(4, dtype=torch.long))
    with pytest.raises(ValueError, match="graph_attr is missing"):
        m(d)
    assert m.graph_concat_projector is None
    # 1-D and 2-D forms are accepted
    assert m._graph_attr(hb.Batch(graph_attr=torch.ones(6)), 3, torch.zeros(1)).shape == (3, 2)
    assert m._graph_attr(hb.Batch(graph_attr=torch.ones(3, 2)), 3, torch.zeros(1)).shape == (3, 2)


@pytest.mark.parametrize("mpnn_type", ["EGNN", "PAINN", "SchNet", "CGCNN", "GAT", "SAGE"])
def test_other_stacks_refuse_conditioning_via_create_model_and_create_model_config(mpnn_type):
    kw = dict(input_dim=1, hidden_dim=8, output_dim=[1], output_type=["graph"], output_heads={"graph": {"num_sharedlayers": 1,
              "dim_sharedlayers": 4, "num_headlayers": 1, "dim_headlayers": [4]}}, task_weights=[1.0], num_conv_layers=1,
              num_radial=4, radius=3.0, num_gaussians=4, num_filters=8, use_gpu=False)
    with pytest.raises(ValueError, match="graph_attr conditioning is not implemented"):
        hb.create_model(mpnn_type=mpnn_type, use_graph_attr_conditioning=True, **kw)
    arch = dict(mpnn_type=mpnn_type, input_dim=1, hidden_dim=8, output_dim=[1], output_type=["graph"],
                output_heads=kw["output_heads"], task_weights=[1.0], num_conv_layers=1, num_radial=4, radius=3.0, num_gaussians=4,
                num_filters=8, use_graph_attr_conditioning=True)
    with pytest.raises(ValueError, match="graph_attr conditioning is not implemented"):
        hb.create_model_config({"Architecture": arch, "Training": {}}, use_gpu=False)


def test_create_model_config_forwards_the_conditioning_keys():
    arch = dict(mpnn_type="MACE", **{k: v for k, v in MACE_KW.items() if k not in ("output_heads", "task_weights", "loss_function_type")},
                output_heads=MACE_KW["output_heads"], task_weights=[1.0, 1.0], use_graph_attr_conditioning=True)
    m = hb.create_model_config({"Architecture": arch, "Training": {"loss_function_type": "mae"}}, use_gpu=False)
    assert m.use_graph_attr_conditioning and m.graph_attr_conditioning_mode == "concat_node"      # the config's default mode
    arch["graph_attr_conditioning_mode"] = "FiLM"
    m = hb.create_model_config({"Architecture": arch, "Training": {"loss_function_type": "mae"}}, use_gpu=False)
    assert m.graph_attr_conditioning_mode == "film"


def test_flat_adamw_refuses_a_model_whose_conditioning_modules_do_not_exist_yet():
    m = _engine(dict(use_graph_attr_conditioning=True, graph_attr_conditioning_mode="film"))
    with pytest.raises(ValueError, match="run one forward"):
        hb.FlatAdamW(m)
    m = hb.create_model(mpnn_type="MACE", use_gpu=False, enable_interatomic_potential=True, energy_weight=1.0, force_weight=1.0,
                        use_graph_attr_conditioning=True, graph_attr_conditioning_mode="concat_node",
                        **dict(MACE_KW, output_dim=[1], output_type=["node"], task_weights=[1.0]))
    with pytest.raises(ValueError, match="run one forward"):
        hb.FlatAdamW(m)
