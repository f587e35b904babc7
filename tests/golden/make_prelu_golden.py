"""Generate tests/golden/models_prelu.pt by running the REFERENCE's own Base.py, stack files and MACE blocks with
activation_function "prelu" (hydragnn/utils/model/model.py:30-46: one ``torch.nn.PReLU()`` that Base.__init__ builds once and
every head layer, feature layer, conv-type node head, MACE decoder and FiLM conditioner shares) on the stubs of make_golden.py and
the restated third-party convs.  Run where the reference checkout is (record.REF); the tests never read it.

    python tests/golden/make_prelu_golden.py      # writes models_prelu.pt, nothing else

Stack cases store what ``record_case`` stores (seeded state dict in the reference's key order, eval and train-mode predictions,
the loss, every parameter gradient -- the shared slope's under the first name ``named_parameters`` gives it -- and the BatchNorm
statistics afterwards), plus ``keys``, the full state-dict key list.  The slope is set to ``SLOPE`` before recording in the cases
named ``*_slope``, so the negative branch is exercised away from the default 0.25 as well.  Cases:

* ``pna_ci_multihead``: the architecture of the reference's tests/inputs/ci_multihead.json (BatchNorm feature layers);
* ``egnn_graph_node``: EGNN with a graph head and an ``mlp`` node head;
* ``egnn_two_branches``: EGNN with two graph-head branches chosen by ``dataset_name`` (the engine's grouped decode);
* ``painn_mlp_per_node``: PaiNN with an ``mlp_per_node`` head;
* ``pna_conv_head_slope``: a conv-type node head (``act(bn(conv))`` at every head layer), slope -0.3;
* ``pna_gps``: PNA inside GPS;
* ``sage_graph_slope``: SAGE with a graph head, slope -0.3;
* ``egnn_gnll``: EGNN with graph and node heads under GaussianNLLLoss (means, then variances);
* ``mace`` / ``mace_film``: MACE with graph and ``mlp`` node heads, the second FiLM-conditioned (its graph_conditioner, created
  at the first forward, holds the same PReLU).  Recorded as the MACE goldens are: eval mode, the objective
  sum(graph) + sum(node^2), its position gradient and every parameter gradient.

``errors`` holds what the reference raises (``refusal``) with "prelu"; it is empty when every case runs.
"""
import torch

import make_golden as mg
from make_pna_golden import install_pna_stubs
from make_sage_mfc_golden import install_sage_mfc_stubs
from record import HERE, add_edge_and_pe, degree_histogram, pna_batch, record_case, refusal, save, t2d, targets

ACT = "prelu"
SLOPE = -0.3
GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 7]}
CI_GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 10, "num_headlayers": 2, "dim_headlayers": [10, 10]}
CI_NODE = {"num_headlayers": 2, "dim_headlayers": [10, 10], "type": "mlp"}
NODE = {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}
PER_NODE = {"num_headlayers": 2, "dim_headlayers": [7, 5], "type": "mlp_per_node"}
CONV = {"num_headlayers": 2, "dim_headlayers": [10, 6], "type": "conv"}


def heads(graph=None, node=None, branches=1):
    out = {}
    if graph is not None:
        out["graph"] = [{"type": "branch-%d" % i, "architecture": graph} for i in range(branches)]
    if node is not None:
        out["node"] = [{"type": "branch-0", "architecture": node}]
    return out


class Flat:
    """A mean-and-variance model seen as one returning a list: the means of every head, then their variances."""

    def __init__(self, m):
        self.m = m

    def __getattr__(self, name):
        return getattr(self.m, name)

    def __str__(self):
        return str(self.m)

    def __call__(self, data):
        mean, var = self.m(data)
        return list(mean) + list(var)

    def loss(self, pred, value, head_index):
        k = len(pred) // 2
        return self.m.loss((pred[:k], pred[k:]), value, head_index)


def set_slope(m, value):
    with torch.no_grad():
        m.activation_function.weight.fill_(value)


def record(m, b, kinds, gen, cfg, slope=None, dims=None):
    assert isinstance(m.activation_function, torch.nn.PReLU)
    if slope is not None:
        set_slope(m, slope)
    if dims is None:
        rec = record_case(m, b, *targets(b, kinds, gen), cfg=dict(cfg, activation_function=ACT))
    else:                                                                   # GaussianNLLLoss: every head is d wide
        from make_gnll_golden import targets as nll_targets
        rec = record_case(Flat(m), b, *nll_targets(b, kinds, dims, gen), cfg=dict(cfg, activation_function=ACT,
                                                                                   loss_function_type="GaussianNLLLoss"))
    rec["keys"] = list(rec["state"])
    rec["slope"] = slope
    return rec


def pna(mod, b, input_dim, hidden, otype, odim, hd, weights, use_gps=False, loss="mse"):
    torch.manual_seed(0)
    return mod.PNAStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", degree_histogram(b), None,
                        input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                        4 if use_gps else 0, otype, hd, ACT, loss, False, loss_weights=weights, freeze_conv=False,
                        initial_bias=None, num_conv_layers=2, num_nodes=None, graph_pooling="mean")


def egnn(egcl, input_dim, hidden, otype, odim, hd, loss="mse"):
    torch.manual_seed(0)
    return egcl.EGCLStack("inv_node_feat, equiv_node_feat, edge_index, edge_attr, edge_shifts", "", None,
                          input_dim, hidden, odim, 0, "", "", 0, otype, hd, ACT, loss, False, max_neighbours=None,
                          loss_weights=[1.0] * len(otype), freeze_conv=False, initial_bias=None, num_conv_layers=2,
                          num_nodes=None, graph_pooling="mean")


def make_base_stacks(gen, out):
    pmod = install_pna_stubs()
    import sys
    egcl, painn = sys.modules["hydragnn.models.EGCLStack"], sys.modules["hydragnn.models.PAINNStack"]
    pcfg = dict(input_dim=1, hidden_dim=8, num_conv_layers=2, edge_dim=None, graph_pooling="mean", gps=False)

    b = pna_batch(gen, [7, 5, 9, 6], 1)
    otype, odim, hd = ["graph", "node", "node", "node"], [1, 1, 1, 1], heads(CI_GRAPH, CI_NODE)
    m = pna(pmod, b, 1, 8, otype, odim, hd, [20.0, 1.0, 1.0, 1.0])
    rec = record(m, b, otype, gen, dict(pcfg, output_type=otype, output_dim=odim, output_heads=hd))
    rec["deg"], rec["task_weights"] = degree_histogram(b), [20.0, 1.0, 1.0, 1.0]
    out["pna_ci_multihead"] = rec

    b = pna_batch(gen, [7, 5, 9, 6], 1)
    otype, odim, hd = ["node"], [1], heads(node=CONV)
    m = pna(pmod, b, 1, 8, otype, odim, hd, [1.0])
    rec = record(m, b, otype, gen, dict(pcfg, output_type=otype, output_dim=odim, output_heads=hd), slope=SLOPE)
    rec["deg"] = degree_histogram(b)
    out["pna_conv_head_slope"] = rec

    b = add_edge_and_pe(pna_batch(gen, [7, 5, 9, 6], 2), gen, None, None, True)
    otype, odim, hd = ["graph"], [1], heads(GRAPH)
    m = pna(pmod, b, 2, 16, otype, odim, hd, [1.0], use_gps=True)
    rec = record(m, b, otype, gen, dict(pcfg, input_dim=2, hidden_dim=16, gps=True, output_type=otype, output_dim=odim,
                                        output_heads=hd))
    rec["deg"] = degree_histogram(b)
    out["pna_gps"] = rec

    ecfg = dict(input_dim=1, hidden_dim=12, num_conv_layers=2, edge_dim=None, graph_pooling="mean", gps=False)
    b = mg.toy_batch(gen, [6, 5, 8, 3], 4.0)
    otype, odim, hd = ["graph", "node"], [1, 1], heads(GRAPH, NODE)
    out["egnn_graph_node"] = record(egnn(egcl, 1, 12, otype, odim, hd), b, otype, gen,
                                    dict(ecfg, output_type=otype, output_dim=odim, output_heads=hd))

    b = mg.toy_batch(gen, [6, 5, 8, 3, 7, 4], 4.0)
    b.dataset_name = torch.tensor([[0], [1], [1], [0], [1], [0]])
    hd = heads(GRAPH, branches=2)
    out["egnn_two_branches"] = record(egnn(egcl, 1, 12, ["graph"], [1], hd), b, ["graph"], gen,
                                      dict(ecfg, output_type=["graph"], output_dim=[1], output_heads=hd))

    b = mg.toy_batch(gen, [6, 5, 8, 3], 4.0)
    otype, odim, hd = ["graph", "node"], [1, 2], heads(GRAPH, NODE)
    out["egnn_gnll"] = record(egnn(egcl, 1, 12, otype, odim, hd, loss="GaussianNLLLoss"), b, otype, gen,
                              dict(ecfg, output_type=otype, output_dim=odim, output_heads=hd), dims=odim)

    b = mg.toy_batch(gen, [6, 6, 6], 5.0)
    hd = heads(node=PER_NODE)
    torch.manual_seed(0)
    m = painn.PAINNStack("inv_node_feat, equiv_node_feat, edge_index, diff, dist", "inv_node_feat, equiv_node_feat, edge_index, diff, dist",
                         None, 5, 7.0, 1, 12, [2], 0, "", "", 0, ["node"], hd, ACT, "mse", False, loss_weights=[1.0],
                         freeze_conv=False, num_conv_layers=2, num_nodes=6, graph_pooling="mean")
    rec = record_case(m, b, *_node_targets(b, 2, gen), cfg=dict(input_dim=1, hidden_dim=12, num_conv_layers=2, output_type=["node"],
                                                                 output_dim=[2], output_heads=hd, num_nodes=6, num_radial=5,
                                                                 radius=7.0, edge_dim=None, graph_pooling="mean", gps=False,
                                                                 activation_function=ACT))
    rec["keys"], rec["slope"] = list(rec["state"]), None
    out["painn_mlp_per_node"] = rec


def _node_targets(b, d, gen):
    n = b.x.shape[0]
    return torch.randn(n * d, generator=gen), [torch.arange(n * d)]


def make_sage(gen, out):
    sage, _ = install_sage_mfc_stubs()
    b = pna_batch(gen, [7, 5, 9, 6], 3)
    hd = heads(GRAPH)
    torch.manual_seed(0)
    m = sage.SAGEStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", 3, 8, [1], 0, None, None, 0,
                       ["graph"], hd, ACT, "mse", False, loss_weights=[1.0], freeze_conv=False, num_conv_layers=2,
                       num_nodes=None, graph_pooling="mean")
    out["sage_graph_slope"] = record(m, b, ["graph"], gen, dict(input_dim=3, hidden_dim=8, num_conv_layers=2, output_type=["graph"],
                                                                 output_dim=[1], graph_pooling="mean", gps=False, output_heads=hd,
                                                                 num_nodes=None, initial_bias=None), slope=SLOPE)


MACE_HEADS = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                               "dim_headlayers": [10, 6]}}],
              "node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}}]}


def make_mace(gen, out, errors):
    mg.install_stubs()
    mace = mg.install_mace_stubs()
    for name, mode in (("mace", None), ("mace_film", "film")):
        b = mg.toy_batch(gen, [7, 9, 5], 3.5, input_dim=1)
        if mode:
            b.graph_attr = torch.randn(3, 2, generator=gen)
        cond = dict(use_graph_attr_conditioning=True, graph_attr_conditioning_mode=mode) if mode else {}

        def build():
            torch.manual_seed(0)
            return mace.MACEStack("node_attributes, equiv_node_feat, inv_node_feat, edge_attributes, edge_features, edge_index",
                                  "node_attributes, edge_attributes, edge_features, edge_index", 6.0, "bessel", None, 8, None,
                                  2, 1, 10.0, 5, 2, 1, 8, [1, 3], 0, "", "", 0, ["graph", "node"], MACE_HEADS,
                                  ACT, "mae", None, loss_weights=[1.0, 1.0], freeze_conv=False, initial_bias=None,
                                  num_conv_layers=2, num_nodes=9, graph_pooling="mean", **cond)
        inp = t2d(b)

        def run():
            m = build()
            m.eval()
            pos0 = b.pos.clone().requires_grad_(True)
            b.pos = pos0
            torch.manual_seed(1234)                     # the lazy conditioning modules draw from this state at the first forward
            try:
                pred = m(b)
            finally:
                b.pos = inp["pos"]
            obj = pred[0].sum() + pred[1].pow(2).sum()
            forces = torch.autograd.grad(obj, pos0, retain_graph=True)[0]
            grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
            state = {k: v.clone() for k, v in m.state_dict().items()}           # after the forward: the conditioner included
            out[name] = {"state": state, "keys": list(state), "inputs": inp, "pred": [p.detach() for p in pred],
                         "dobj_dpos": forces.detach(),
                         "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)},
                         "cfg": dict(max_ell=2, node_max_ell=1, correlation=2, num_conv_layers=2, hidden_dim=8,
                                     activation_function=ACT, **cond)}
        err = refusal(run)
        if err is not None:
            errors[name] = err


def main():
    gen = torch.Generator().manual_seed(20261019)
    out, errors = {}, {}
    make_base_stacks(gen, out)
    make_sage(gen, out)
    make_mace(gen, out, errors)
    out["errors"] = errors
    save(out, HERE + "/models_prelu.pt")


if __name__ == "__main__":
    main()
