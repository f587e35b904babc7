"""fp64 CPU restatement of the reference's mean-and-variance heads (loss_function_type "GaussianNLLLoss", hydragnn/models/Base.py:
109-111 var_output, 565-583 and 634-664 the 2 d-wide last layers, 764-846 the (outputs, outputs_var) return, 848-906 the loss),
on top of the oracle stacks of oracle/.  tests/golden/models_gnll.pt pins it against the reference's code.

``with_variance(cls)`` turns an oracle stack class into its GaussianNLL form without touching the stack: every head is built and
run at width 2 d (``head_dims`` doubled while ``_multihead`` and ``forward`` run, so the graph heads, ``mlp`` / ``mlp_per_node``
heads, conv-type node heads and their BatchNorms, single- and multi-branch, are all the stack's own code), each head's output o
is split into the mean o[:, :d] and the variance o[:, d:] ** 2, and the loss is ``torch.nn.GaussianNLLLoss()`` per head, weighted
as in ``loss_hpweighted``.  Also here: what the GaussianNLL test modules share (the cases, their keyword arguments, ``Flat``).
"""
import torch

from oracle.base import OracleModel
from oracle.cgcnn import CGCNNStackOracle
from oracle.pna import PNAStackOracle

CASES = ["pna_ci_multihead", "pna_conv_head", "pna_gps", "egnn_initial_bias", "egnn_two_branches", "egnn_clamped",
         "painn_mlp_per_node", "cgcnn_graph"]
GPS = dict(pe_dim=4, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)


class _VarHeads:
    def __init__(self, *args, loss_function_type="GaussianNLLLoss", **kw):
        assert loss_function_type == "GaussianNLLLoss"
        super().__init__(*args, loss_function_type="mse", **kw)         # the stack's own loss table stops at rmse
        self.var_output, self.loss_function = 1, torch.nn.GaussianNLLLoss()

    def _wide(self, fn):
        dims = self.head_dims
        self.head_dims = [2 * d for d in dims]
        try:
            return fn()
        finally:
            self.head_dims = dims

    def _multihead(self):
        self._wide(super()._multihead)

    def forward(self, data):
        outs = self._wide(lambda: super(_VarHeads, self).forward(data))
        return [o[:, :d] for o, d in zip(outs, self.head_dims)], [o[:, d:] ** 2 for o, d in zip(outs, self.head_dims)]

    def loss(self, pred, value, head_index):
        mean, var = pred
        tot, tasks = 0, []
        for ih in range(self.num_heads):
            tgt = value[head_index[ih]].reshape(mean[ih].shape).to(mean[ih].dtype)
            li = self.loss_function(mean[ih], tgt, var[ih])
            tot = tot + li * self.loss_weights[ih]
            tasks.append(li)
        return tot, tasks


def with_variance(cls):
    return type("Var" + cls.__name__, (_VarHeads, cls), {})


STACKS = {"PNA": with_variance(PNAStackOracle), "CGCNN": with_variance(CGCNNStackOracle)}
VarOracleModel = with_variance(OracleModel)


def mpnn_type(name):
    return {"pna": "PNA", "egnn": "EGNN", "painn": "PAINN", "cgcnn": "CGCNN"}[name.split("_")[0]]


def case_kwargs(name, c):
    """create_model keyword arguments of a case of models_gnll.pt."""
    cfg = dict(c["cfg"])
    if cfg.pop("gps"):
        cfg.update(GPS)
    if "deg" in c:
        cfg["pna_deg"] = c["deg"]
    return dict(cfg, mpnn_type=mpnn_type(name), task_weights=c.get("task_weights", [1.0] * len(cfg["output_type"])))


def oracle_of(name, c):
    """The variance-head oracle of a case with its state loaded strictly, in fp64."""
    kw = case_kwargs(name, c)
    kw.pop("initial_bias", None)
    t = kw.pop("mpnn_type")
    m = STACKS[t](**kw, dropout=0.0) if t in STACKS else VarOracleModel(t, **kw, dropout=0.0)
    m.load_state_dict(c["state"], strict=True)
    return m.double()


class Flat:
    """A mean-and-variance model seen as one returning the list the golden stores: the means of every head, then their
    variances."""

    def __init__(self, m):
        self.m = m

    def __getattr__(self, name):
        return getattr(self.m, name)

    def __call__(self, data):
        mean, var = self.m(data)
        return list(mean) + list(var)

    def loss(self, pred, value, head_index):
        k = len(pred) // 2
        return self.m.loss((pred[:k], pred[k:]), value, head_index)
