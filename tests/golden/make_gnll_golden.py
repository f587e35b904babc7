"""Generate tests/golden/models_gnll.pt by running the REFERENCE's own Base.py and stack files with loss_function_type
"GaussianNLLLoss" (mean-and-variance heads, hydragnn/models/Base.py:109-111, 634-664, 565-583, 764-846, 848-906) on the stubs of
make_golden.py and the restated third-party convs (oracle/pna.py, oracle/cgcnn.py, oracle/gat.py).  Run in the build container
only; the reference tree does not exist on the GPU machines.

    python tests/golden/make_gnll_golden.py      # writes models_gnll.pt, nothing else

Every case stores what ``record_case`` stores.  A GaussianNLL model returns (outputs, outputs_var), so the model is recorded
through ``Flat``, which shows the recorder one list: the means of every head, then the variances.  Cases:

* ``pna_ci_multihead``: the architecture of the reference's tests/inputs/ci_multihead.json (one graph head, three ``mlp`` node
  heads, hidden 8, task weights [20, 1, 1, 1]);
* ``egnn_initial_bias``: EGNN, one graph head, ``initial_bias`` 0.5.  The reference's ``Base._set_bias`` fails on the head's
  branch dict (the KeyError is recorded under ``errors``), so the maker fills the last bias of the branch, all 2 d entries, as
  the engine's Base does;
* ``egnn_two_branches``: EGNN with two graph-head branches chosen by ``dataset_name`` (the multibranch GFM shape);
* ``painn_mlp_per_node``: PaiNN with an ``mlp_per_node`` head of width 2;
* ``pna_conv_head``: a ``conv`` node head of width 2 built by ``Base._init_node_conv``;
* ``pna_gps``: PNA inside GPS;
* ``cgcnn_graph``: CGCNN with a graph head;
* ``egnn_clamped``: the variance rows of every head's last layer set to zero, so every variance is clamped to eps.

``errors`` holds what the reference raises (``refusal``) for MACE, an interatomic potential, GAT and CGCNN conv-type node heads
under GaussianNLLLoss, and for ``initial_bias`` on a graph head.
"""
import sys
import types

import torch

import make_golden as mg
from make_pna_golden import install_pna_stubs
from record import HERE, REF, add_edge_and_pe, degree_histogram, pna_batch, record_case, refusal, save

NLL = "GaussianNLLLoss"
GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2, "dim_headlayers": [10, 7]}
CI_GRAPH = {"num_sharedlayers": 2, "dim_sharedlayers": 10, "num_headlayers": 2, "dim_headlayers": [10, 10]}
CI_NODE = {"num_headlayers": 2, "dim_headlayers": [10, 10], "type": "mlp"}
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


def targets(b, kinds, dims, gen):
    """(value, head_index) as Base.loss reads them: one flat vector, one index tensor of rows x dim entries per head."""
    g, n = int(b.batch.max()) + 1, b.x.shape[0]
    vals, idx, off = [], [], 0
    for k, d in zip(kinds, dims):
        size = (g if k == "graph" else n) * d
        vals.append(torch.randn(size, generator=gen))
        idx.append(torch.arange(off, off + size))
        off += size
    return torch.cat(vals), idx


def record(m, b, kinds, dims, gen, cfg):
    rec = record_case(Flat(m), b, *targets(b, kinds, dims, gen), cfg=dict(cfg, loss_function_type=NLL))
    rec.pop("str")
    return rec


def pna(mod, b, input_dim, hidden, layers, otype, odim, hd, weights, use_gps=False):
    torch.manual_seed(0)
    return mod.PNAStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", degree_histogram(b), None,
                        input_dim, hidden, odim, 4 if use_gps else 0, "GPS" if use_gps else None, "multihead" if use_gps else None,
                        4 if use_gps else 0, otype, hd, "relu", NLL, False, loss_weights=weights, freeze_conv=False,
                        initial_bias=None, num_conv_layers=layers, num_nodes=None, graph_pooling="mean")


def egnn(egcl, input_dim, hidden, otype, odim, hd, initial_bias=None):
    torch.manual_seed(0)
    return egcl.EGCLStack("inv_node_feat, equiv_node_feat, edge_index, edge_attr, edge_shifts", "", None,
                          input_dim, hidden, odim, 0, "", "", 0, otype, hd, "relu", NLL, False, max_neighbours=None,
                          loss_weights=[1.0] * len(otype), freeze_conv=False, initial_bias=initial_bias, num_conv_layers=2,
                          num_nodes=None, graph_pooling="mean")


def make_pna_egnn_painn(gen, out, errors):
    pmod = install_pna_stubs()
    egcl, painn = sys.modules["hydragnn.models.EGCLStack"], sys.modules["hydragnn.models.PAINNStack"]

    b = pna_batch(gen, [7, 5, 9, 6], 1)
    otype, odim, hd = ["graph", "node", "node", "node"], [1, 1, 1, 1], heads(CI_GRAPH, CI_NODE)
    m = pna(pmod, b, 1, 8, 2, otype, odim, hd, [20.0, 1.0, 1.0, 1.0])
    rec = record(m, b, otype, odim, gen, dict(input_dim=1, hidden_dim=8, num_conv_layers=2, output_type=otype, output_dim=odim,
                                              edge_dim=None, graph_pooling="mean", gps=False, output_heads=hd))
    rec["deg"], rec["task_weights"] = degree_histogram(b), [20.0, 1.0, 1.0, 1.0]
    out["pna_ci_multihead"] = rec

    b = pna_batch(gen, [7, 5, 9, 6], 1)
    otype, odim, hd = ["node"], [2], heads(node=CONV)
    m = pna(pmod, b, 1, 8, 2, otype, odim, hd, [1.0])
    rec = record(m, b, otype, odim, gen, dict(input_dim=1, hidden_dim=8, num_conv_layers=2, output_type=otype, output_dim=odim,
                                              edge_dim=None, graph_pooling="mean", gps=False, output_heads=hd))
    rec["deg"] = degree_histogram(b)
    out["pna_conv_head"] = rec

    b = add_edge_and_pe(pna_batch(gen, [7, 5, 9, 6], 2), gen, None, None, True)
    otype, odim, hd = ["graph"], [1], heads(GRAPH)
    m = pna(pmod, b, 2, 16, 2, otype, odim, hd, [1.0], use_gps=True)
    rec = record(m, b, otype, odim, gen, dict(input_dim=2, hidden_dim=16, num_conv_layers=2, output_type=otype, output_dim=odim,
                                              edge_dim=None, graph_pooling="mean", gps=True, output_heads=hd))
    rec["deg"] = degree_histogram(b)
    out["pna_gps"] = rec

    ecfg = dict(input_dim=1, hidden_dim=12, num_conv_layers=2, edge_dim=None, graph_pooling="mean", gps=False)
    b = mg.toy_batch(gen, [6, 5, 8, 3], 4.0)
    hd = heads(GRAPH)
    errors["initial_bias_graph"] = refusal(lambda: egnn(egcl, 1, 12, ["graph"], [1], hd, initial_bias=0.5))
    m = egnn(egcl, 1, 12, ["graph"], [1], hd)
    m.heads_NN[0]["branch-0"][-1].bias.data.fill_(0.5)            # what the engine's Base fills: every graph branch's last bias
    out["egnn_initial_bias"] = record(m, b, ["graph"], [1], gen, dict(ecfg, output_type=["graph"], output_dim=[1], output_heads=hd,
                                                                       initial_bias=0.5))

    b = mg.toy_batch(gen, [6, 5, 8, 3, 7, 4], 4.0)
    b.dataset_name = torch.tensor([[0], [1], [1], [0], [1], [0]])
    hd = heads(GRAPH, branches=2)
    m = egnn(egcl, 1, 12, ["graph"], [1], hd)
    out["egnn_two_branches"] = record(m, b, ["graph"], [1], gen, dict(ecfg, output_type=["graph"], output_dim=[1], output_heads=hd))

    b = mg.toy_batch(gen, [6, 5, 8, 3], 4.0)
    otype, odim, hd = ["graph", "node"], [1, 2], heads(GRAPH, {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"})
    m = egnn(egcl, 1, 12, otype, odim, hd)
    with torch.no_grad():
        for head, d in zip(m.heads_NN, odim):
            last = head["branch-0"][-1] if otype[0] == "graph" and head is m.heads_NN[0] else head["branch-0"].mlp[0][-1]
            last.weight[d:] = 0.0
            last.bias[d:] = 0.0
    rec = record(m, b, otype, odim, gen, dict(ecfg, output_type=otype, output_dim=odim, output_heads=hd))
    rec["var_rows_zeroed"] = True
    out["egnn_clamped"] = rec

    b = mg.toy_batch(gen, [6, 6, 6], 5.0)
    hd = heads(node=PER_NODE)
    torch.manual_seed(0)
    m = painn.PAINNStack("inv_node_feat, equiv_node_feat, edge_index, diff, dist", "inv_node_feat, equiv_node_feat, edge_index, diff, dist",
                         None, 5, 7.0, 1, 12, [2], 0, "", "", 0, ["node"], hd, "relu", NLL, False, loss_weights=[1.0],
                         freeze_conv=False, num_conv_layers=2, num_nodes=6, graph_pooling="mean")
    out["painn_mlp_per_node"] = record(m, b, ["node"], [2], gen, dict(input_dim=1, hidden_dim=12, num_conv_layers=2, output_type=["node"],
                                                                      output_dim=[2], output_heads=hd, num_nodes=6, num_radial=5,
                                                                      radius=7.0, edge_dim=None, graph_pooling="mean", gps=False))

    # an interatomic potential: the reference's energy_force_loss on the (outputs, outputs_var) pair of a node-head model
    b = mg.toy_batch(gen, [6, 5], 4.0)
    m = egnn(egcl, 1, 8, ["node"], [1], heads(node={"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}))
    glb = {"torch": torch, "torch_scatter": sys.modules["torch_scatter"]}
    mg._extract(REF + "/hydragnn/models/create.py", ["energy_force_loss"], glb)
    fake = types.SimpleNamespace(num_heads=1, head_type=["node"], model=m, loss_function=m.loss_function,
                                 energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)

    def mlip():
        b.pos.requires_grad_(True)
        glb["energy_force_loss"](fake, m(b), b, create_graph=True)
    errors["mlip"] = refusal(mlip)


def make_cgcnn(gen, out, errors):
    from make_cgcnn_golden import install_cgcnn_stubs
    mod = install_cgcnn_stubs()

    def build(otype, odim, hd):
        torch.manual_seed(0)
        return mod.CGCNNStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", 0, 3, 3, odim, 0, None,
                              None, 0, otype, hd, "relu", NLL, False, loss_weights=[1.0] * len(otype), freeze_conv=False,
                              initial_bias=None, num_conv_layers=2, num_nodes=None, graph_pooling="mean")
    b = pna_batch(gen, [7, 5, 9, 6], 3)
    hd = heads(GRAPH)
    out["cgcnn_graph"] = record(build(["graph"], [1], hd), b, ["graph"], [1], gen,
                                dict(input_dim=3, hidden_dim=3, num_conv_layers=2, output_type=["graph"], output_dim=[1], edge_dim=0,
                                     graph_pooling="mean", gps=False, output_heads=hd))
    errors["cgcnn_conv_head"] = refusal(lambda: build(["node"], [1], heads(node=CONV)))


def make_gat(gen, errors):
    from make_gat_golden import install_gat_stubs
    mod = install_gat_stubs()
    b = pna_batch(gen, [7, 5, 9, 6], 3)

    def run():
        torch.manual_seed(0)
        m = mod.GATStack("inv_node_feat, equiv_node_feat, edge_index", "inv_node_feat, edge_index", 6, 0.05, None, 3, 8, [1], 0,
                         None, None, 0, ["node"], heads(node=CONV), "relu", NLL, False, loss_weights=[1.0], freeze_conv=False,
                         initial_bias=None, num_conv_layers=2, num_nodes=None, graph_pooling="mean")
        m.loss(m(b), *targets(b, ["node"], [1], gen))
    errors["gat_conv_head"] = refusal(run)


def make_mace(gen, errors):
    mace = mg.install_mace_stubs()
    b = mg.toy_batch(gen, [7, 5], 3.5)
    hd = heads(GRAPH, {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"})

    def run():
        torch.manual_seed(0)
        m = mace.MACEStack("node_attributes, equiv_node_feat, inv_node_feat, edge_attributes, edge_features, edge_index",
                           "node_attributes, edge_attributes, edge_features, edge_index", 6.0, "bessel", None, 8, None, 2, 1, 10.0,
                           5, 2, 1, 8, [1, 1], 0, "", "", 0, ["graph", "node"], hd, "relu", NLL, None, loss_weights=[1.0, 1.0],
                           freeze_conv=False, initial_bias=None, num_conv_layers=2, num_nodes=9, graph_pooling="mean")
        m.loss(m(b), *targets(b, ["graph", "node"], [1, 1], gen))
    errors["mace"] = refusal(run)


def main():
    gen = torch.Generator().manual_seed(20261018)
    out, errors = {}, {}
    make_pna_egnn_painn(gen, out, errors)
    make_cgcnn(gen, out, errors)
    make_gat(gen, errors)
    make_mace(gen, errors)
    assert all(errors.values()), errors
    out["errors"] = errors
    save(out, HERE + "/models_gnll.pt")


if __name__ == "__main__":
    main()
