"""CPU tests of MACE's distance transforms (distance_transform "Agnesi" / "Soft"): the covalent-radii table, the engine's and the
fp64 oracle's construction against tests/golden/models_mace_transform.pt (the reference's own MACEStack,
tests/golden/make_mace_transform_golden.py), and the oracle's outputs, forces and gradients against the same golden."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200.covalent_radii import COVALENT_RADII, covalent_radii_tensor
from oracle.mace_transform import MACETransformOracle
from oracle.mlip import MLIPWrapper
from mace_transform_support import load_golden
from stack_support import MACE_KW

TRANSFORM_KEYS = {"Agnesi": ["q", "p", "a", "covalent_radii"], "Soft": ["covalent_radii", "a", "b"]}


def rel_l2(a, b):
    return float((a.detach().double() - b.double()).norm() / b.double().norm().clamp(min=1e-30))


def _golden(golden_dir):
    return load_golden(golden_dir)


def _inner(m):
    return m.model if hasattr(m, "energy_force_loss") else m


def _batch(inputs):
    d = hb.Batch(**{k: (v.clone().double() if v.is_floating_point() else v.clone()) for k, v in inputs.items()})
    d._num_graphs = 3
    d.pos.requires_grad_(True)
    return d


def test_covalent_radii_table():
    assert len(COVALENT_RADII) == 119
    assert COVALENT_RADII[0] == 0.2 and all(r == 0.2 for r in COVALENT_RADII[97:])
    assert all(r != 0.2 for r in COVALENT_RADII[1:97])
    for z, r in [(1, 0.31), (6, 0.76), (8, 0.66), (26, 1.32), (96, 1.69)]:      # H, C (sp3), O, Fe (low spin), Cm
        assert COVALENT_RADII[z] == r
    t = covalent_radii_tensor()
    assert t.dtype == torch.float32 and t.shape == (119,)


def test_engine_construction_matches_the_reference_own_code_golden(golden_dir):
    """Keys, order, dtypes and values: the transform's buffers sit between bessel_fn and cutoff_fn."""
    for name, c in _golden(golden_dir).items():
        m = _inner(hb.create_model(mpnn_type="MACE", use_gpu=False, **dict(MACE_KW, **c["cfg"])))
        se, params = m.state_dict(), dict(m.named_parameters())
        assert list(se.keys()) == list(c["state"].keys()), name
        for k, v in se.items():
            ref = c["state"][k]
            assert v.dtype == ref.dtype and v.shape == ref.shape, (name, k)
            if k in params or ".distance_transform." in k:
                assert torch.equal(v, ref), (name, k)
            else:
                assert torch.allclose(v, ref, atol=1e-6), (name, k)
        kind = c["cfg"]["distance_transform"]
        keys = [k for k in se if k.startswith("radial_embedding.")]
        i = keys.index("radial_embedding.cutoff_fn.p")
        assert keys[i - len(TRANSFORM_KEYS[kind]):i] == ["radial_embedding.distance_transform." + b for b in TRANSFORM_KEYS[kind]]
        assert not any("distance_transform" in k for k in params)
        assert torch.equal(se["radial_embedding.distance_transform.covalent_radii"], covalent_radii_tensor())


@pytest.mark.parametrize("other", [None, "None", "none", "agnesi", "gaussian"])
def test_no_transform_state_dict_is_unchanged(other):
    """Anything but the exact strings "Agnesi" and "Soft" means no transform, silently (blocks.py:154-158)."""
    torch.manual_seed(0)
    base = hb.create_model(mpnn_type="MACE", use_gpu=False, **MACE_KW)
    torch.manual_seed(0)
    m = hb.create_model(mpnn_type="MACE", use_gpu=False, **dict(MACE_KW, distance_transform=other))
    assert m.distance_transform is None
    sa, sb = base.state_dict(), m.state_dict()
    assert list(sa) == list(sb) and not any("distance_transform" in k for k in sb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k


def test_no_transform_state_dict_matches_the_mace_golden(golden_dir):
    c = torch.load(golden_dir + "/models_mace.pt")["mace_l2_nu2"]
    m = hb.create_model(mpnn_type="MACE", use_gpu=False, **dict(MACE_KW, **c["cfg"]))
    assert list(m.state_dict().keys()) == list(c["state"].keys())


def test_oracle_construction_matches_the_golden(golden_dir):
    for name, c in _golden(golden_dir).items():
        torch.manual_seed(0)
        sd = MACETransformOracle(**dict(MACE_KW, **c["cfg"])).state_dict()
        assert list(sd.keys()) == list(c["state"].keys()), name
        for k, v in sd.items():
            assert v.dtype == c["state"][k].dtype and torch.equal(v, c["state"][k]), (name, k)


def test_oracle_matches_the_reference_own_code_golden(golden_dir):
    for name, c in _golden(golden_dir).items():
        if "forces" in c:
            continue
        torch.manual_seed(0)
        m = MACETransformOracle(**dict(MACE_KW, **c["cfg"]))
        m.eval()
        d = _batch(c["inputs"])
        m = m.double()
        pred = m(d)
        # rel-L2 (fp64 against the reference's fp32): the Chebyshev basis of t spans many orders of magnitude
        for p, q in zip(pred, c["pred"]):
            assert rel_l2(p, q) < 1e-5, (name, rel_l2(p, q))
        obj = pred[0].sum() + pred[1].pow(2).sum()
        f, = torch.autograd.grad(obj, d.pos, retain_graph=True)
        assert rel_l2(f, c["dobj_dpos"]) < 1e-4, (name, rel_l2(f, c["dobj_dpos"]))
        grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), (name, n)
            if gr is not None and float(ref.abs().max()) > 0:
                assert rel_l2(gr, ref) < 1e-4, (name, n, rel_l2(gr, ref))


def test_oracle_mlip_matches_the_reference_own_code_golden(golden_dir):
    """Energy, forces and the force loss's parameter gradients (the double backward through the transform)."""
    cases = [(n, c) for n, c in _golden(golden_dir).items() if "forces" in c]
    assert len(cases) == 2
    for name, c in cases:
        torch.manual_seed(0)
        m = MACETransformOracle(**dict(MACE_KW, **c["cfg"]))
        m.eval()
        w = MLIPWrapper(m.double(), 1.0, 1.0, 1.0)
        d = _batch(c["inputs"])
        pred = w(d)
        assert rel_l2(pred[0], c["pred"][0]) < 1e-5
        energy = pred[0].sum()
        f = -torch.autograd.grad(energy, d.pos, retain_graph=True)[0]
        assert rel_l2(f, c["forces"]) < 1e-4, (name, rel_l2(f, c["forces"]))
        tot, tasks = w.energy_force_loss(pred, d)
        torch.testing.assert_close(tot.double(), c["loss"].double(), rtol=1e-5, atol=1e-6)
        for a, b in zip(tasks, c["tasks"]):
            torch.testing.assert_close(a.double(), b.double(), rtol=1e-5, atol=1e-6)
        grads = torch.autograd.grad(tot, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), (name, n)
            if gr is not None and float(ref.abs().max()) > 0:
                assert rel_l2(gr, ref) < 1e-4, (name, n, rel_l2(gr, ref))


def test_transforms_reach_the_output(golden_dir):
    """Changing a radius or a transform parameter changes the oracle's output (the buffers are read, not constants)."""
    c = _golden(golden_dir)["agnesi_bessel"]
    torch.manual_seed(0)
    m = MACETransformOracle(**dict(MACE_KW, **c["cfg"])).double()
    d = _batch(c["inputs"])
    base = m(d)[0].detach()
    with torch.no_grad():
        m.radial_embedding.distance_transform.covalent_radii[6] += 0.3
    assert float((m(d)[0].detach() - base).abs().max()) > 1e-6


def test_gfm_mace_config_with_agnesi_builds():
    """The GFM MACE architecture plus distance_transform "Agnesi" through create_model_config (the search space's draw)."""
    from hydragnn_b200.synthetic import ARCH
    arch = {k: v for k, v in ARCH["gfm_mace"].items() if k not in ("loss_function_type",)}
    arch["distance_transform"] = "Agnesi"
    cfg = {"Architecture": arch, "Training": {"loss_function_type": "mae"}}
    m = hb.create_model_config(cfg, use_gpu=False)
    inner = _inner(m)
    assert inner.distance_transform == "Agnesi"
    assert "radial_embedding.distance_transform.covalent_radii" in inner.state_dict()
