"""CPU tests of MACE with edge attributes (edge_dim > 0): the fp64 restatement (oracle/mace.py) against
tests/golden/models_mace_edge.pt, which comes from the reference's own MACEStack (tests/golden/make_mace_edge_golden.py),
and the engine's initialisation against the same golden."""
import pytest
import torch

import hydragnn_b200 as hb
from hydragnn_b200 import padded
from oracle.mace import MACEOracle
from stack_support import MACE_KW, mace_batch, random_rotation


def _golden(golden_dir):
    return torch.load(golden_dir + "/models_mace_edge.pt")


def test_edge_oracle_matches_the_reference_own_code_golden(golden_dir):
    for name, c in _golden(golden_dir).items():
        torch.manual_seed(0)
        m = MACEOracle(**dict(MACE_KW, **c["cfg"]))
        sd = m.state_dict()
        assert list(sd.keys()) == list(c["state"].keys()), name
        for k, v in sd.items():
            assert torch.equal(v, c["state"][k]), (name, k)
        m.eval()
        d = hb.Batch(**{k: v.clone() for k, v in c["inputs"].items()})
        d._num_graphs = 3
        d.pos.requires_grad_(True)
        pred = m(d)
        for p, q in zip(pred, c["pred"]):
            torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
        obj = pred[0].sum() + pred[1].pow(2).sum()
        f, = torch.autograd.grad(obj, d.pos, retain_graph=True)
        torch.testing.assert_close(f, c["dobj_dpos"], rtol=1e-4, atol=1e-7)
        grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), (name, n)
            if gr is not None:
                torch.testing.assert_close(gr, ref, rtol=1e-4, atol=1e-6 * max(1.0, float(ref.abs().max())))


def test_edge_oracle_with_lengths_is_rotation_invariant():
    torch.manual_seed(0)
    m = MACEOracle(**dict(MACE_KW, edge_dim=1)).double()
    gen = torch.Generator().manual_seed(3)
    d = mace_batch(gen)
    d.edge_attr = (d.pos[d.edge_index[1]] - d.pos[d.edge_index[0]]).norm(dim=1, keepdim=True)
    out = m(d)
    rot = random_rotation(gen)
    d2 = hb.Batch(x=d.x, pos=d.pos @ rot.T, edge_index=d.edge_index, batch=d.batch, edge_attr=d.edge_attr)
    d2._num_graphs = 2
    out2 = m(d2)
    for a, b in zip(out, out2):
        assert float((a - b).abs().max().detach()) < 1e-12
    # the edge attributes reach the output
    d3 = hb.Batch(x=d.x, pos=d.pos, edge_index=d.edge_index, batch=d.batch, edge_attr=d.edge_attr * 1.5)
    d3._num_graphs = 2
    assert float((m(d3)[0] - out[0]).abs().max()) > 1e-6


def test_engine_initialisation_matches_the_reference_own_code_golden(golden_dir):
    for name, c in _golden(golden_dir).items():
        m = hb.create_model(mpnn_type="MACE", use_gpu=False, **dict(MACE_KW, **c["cfg"]))
        se, params = m.state_dict(), dict(m.named_parameters())
        assert list(se.keys()) == list(c["state"].keys()), name
        for k, v in se.items():
            assert v.shape == c["state"][k].shape, (name, k)
            if k in params:             # seeded draws: bit-equal
                assert torch.equal(v, c["state"][k]), (name, k)
            else:                       # coupling tensors and constants, computed (not drawn) by either side
                assert torch.allclose(v, c["state"][k], atol=1e-6), (name, k)


def test_engine_rejects_bad_edge_attr_before_any_kernel():
    m = hb.create_model(mpnn_type="MACE", use_gpu=False, **dict(MACE_KW, edge_dim=2))
    ea = torch.zeros(5, 2)
    assert m._edge_attr(hb.Batch(edge_attr=ea), 5) is not None
    for bad, msg in [(None, "needs data.edge_attr"), (torch.zeros(5, 3), "edge_attr must be"), (torch.zeros(4, 2), "edge_attr must be"),
                     (torch.zeros(5, 2, dtype=torch.float64), "edge_attr must be"), (torch.zeros(5, 2, requires_grad=True), "require grad")]:
        with pytest.raises(ValueError, match=msg):
            m._edge_attr(hb.Batch(edge_attr=bad), 5)


def test_padded_step_refuses_edge_attr_models_with_on_device_neighbour_build():
    m = hb.create_model(mpnn_type="MACE", use_gpu=False, **dict(MACE_KW, edge_dim=1, output_dim=[1], output_type=["graph"],
                                                                 task_weights=[1.0]))
    wrapped = torch.nn.Module()
    wrapped.module = m
    with pytest.raises(ValueError, match="edge_attr"):
        padded.PaddedGraphStep(wrapped, None, hb.Batch(pos=torch.zeros(3, 3)), neighbour_build=(5.0, 8))
