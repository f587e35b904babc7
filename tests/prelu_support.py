"""What the PReLU test modules share: the cases of tests/golden/models_prelu.pt (the reference's own code run with
activation_function "prelu"), their create_model keyword arguments, the engine of a case with its slope set, and the fp64 oracle
of a stack case."""
import hydragnn_b200 as hb
import torch

from gnll_oracle import with_variance
from oracle.base import OracleModel
from oracle.pna import PNAStackOracle
from oracle.sage import SAGEStackOracle
from stack_support import MACE_KW

STACK_CASES = ["pna_ci_multihead", "pna_conv_head_slope", "pna_gps", "egnn_graph_node", "egnn_two_branches", "egnn_gnll",
               "painn_mlp_per_node", "sage_graph_slope"]
MACE_CASES = ["mace", "mace_film"]
GPS = dict(pe_dim=4, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)


def mpnn_type(name):
    return {"pna": "PNA", "egnn": "EGNN", "painn": "PAINN", "sage": "SAGE", "mace": "MACE"}[name.split("_")[0]]


def case_kwargs(name, c):
    """create_model keyword arguments of a case of models_prelu.pt."""
    cfg = dict(c["cfg"])
    if mpnn_type(name) == "MACE":
        return dict(MACE_KW, mpnn_type="MACE", **cfg)
    if cfg.pop("gps"):
        cfg.update(GPS)
    if "deg" in c:
        cfg["pna_deg"] = c["deg"]
    return dict(cfg, mpnn_type=mpnn_type(name), task_weights=c.get("task_weights", [1.0] * len(cfg["output_type"])))


def engine(name, c, use_gpu=False):
    m = hb.create_model(**case_kwargs(name, c), use_gpu=use_gpu)
    if c.get("slope") is not None:
        with torch.no_grad():
            m.activation_function.weight.fill_(c["slope"])
    return m


def oracle_of(name, c):
    """The fp64 oracle of a stack case with the reference's state loaded.  The oracle's heads do not list the shared slope under
    ``MLPNode.activation_function`` as the reference's do; every entry it lacks must be that one slope."""
    kw = case_kwargs(name, c)
    kw.pop("initial_bias", None)
    t = kw.pop("mpnn_type")
    nll = kw.get("loss_function_type") == "GaussianNLLLoss"
    if t == "PNA":
        cls = PNAStackOracle
    elif t == "SAGE":
        cls = SAGEStackOracle
    else:
        cls = None
    if nll:
        m = (with_variance(cls)(**kw, dropout=0.0) if cls else with_variance(OracleModel)(t, **kw, dropout=0.0))
    else:
        kw.pop("loss_function_type", None)
        m = cls(**kw, dropout=0.0) if cls else OracleModel(t, **kw, dropout=0.0)
    own = m.state_dict()
    extra = [k for k in c["state"] if k not in own]
    assert all(k.endswith("activation_function.weight") for k in extra), extra
    slope = c["state"]["activation_function.weight"]
    assert all(torch.equal(c["state"][k], slope) for k in extra)
    m.load_state_dict({k: v for k, v in c["state"].items() if k in own}, strict=True)
    return m.double()
