"""The captured train step rebuilds every index plan cached on its static batch, the hint (edge_index, rowptr, graph_ptr) of a
radius build included: refill copies new edges into the same edge_index tensor, which a kept hint would pair with the old rowptr."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import hydragnn_b200 as hb  # noqa: E402
from hydragnn_b200.synthetic import ARCH, make_samples  # noqa: E402


def _radius_batch(name, g, perm=None, n=9):
    """Edges from the engine's radius build; ``perm`` reorders whole graphs of ``n`` atoms (same counts, different edges)."""
    b = make_samples(name, g, seed=1)
    if perm is not None:
        rows = (perm[:, None] * n + torch.arange(n)[None, :]).reshape(-1)
        b.pos, b.x, b.y = b.pos[rows].contiguous(), b.x[rows].contiguous(), b.y[perm].contiguous()
    b = b.to("cuda")
    b._num_graphs = g
    return hb.get_radius_graph(3.0, 5)(b)                               # r = 3: the edge pattern depends on the geometry


def test_graphed_step_refill_of_a_radius_built_batch_equals_eager():
    name, g = "qm9_painn", 128
    base = _radius_batch(name, g)
    other = _radius_batch(name, g, perm=torch.randperm(g, generator=torch.Generator().manual_seed(3)))
    assert other.edge_index.shape == base.edge_index.shape and not torch.equal(other.edge_index, base.edge_index)
    static = _radius_batch(name, g)                                     # not cloned: it keeps the hint of its radius build
    assert static._hgb_col_sorted[0] is static.edge_index
    m1 = hb.get_distributed_model(hb.create_model(**ARCH[name]))
    m2 = copy.deepcopy(m1)
    o1, o2 = hb.FlatAdamW(m1, lr=1e-3), hb.FlatAdamW(m2, lr=1e-3)
    gs = hb.GraphedTrainStep(m1, o1, static, warmup=2)                  # 2 warm-up steps on `static` (= `base`)
    for _ in range(2):
        hb.train_step(m2, o2, base)
    l_graph = [float(gs.run())]                                         # step 3 on `base`
    l_eager = [float(hb.train_step(m2, o2, base)[0])]
    gs.refill(hb.Batch(x=other.x, pos=other.pos, y=other.y, edge_index=other.edge_index, batch=other.batch))
    l_graph.append(float(gs.run()))                                     # step 4 on `other`: new edges, same shapes
    l_eager.append(float(hb.train_step(m2, o2, other)[0]))
    for a, b in zip(l_graph, l_eager):
        assert abs(a - b) <= 1e-5 * abs(b) + 1e-7, (l_graph, l_eager)
    for p, q in zip(m1.parameters(), m2.parameters()):
        torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-6)
