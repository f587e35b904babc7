"""What the golden makers share: where the reference checkout is, the batches, targets and head tables of the stack goldens, the
record of one model case, of one drop-in dispatch and of one refusal, and ``save``.

The reference checkout is ``HYDRAGNN_REF``, by default ``reference`` next to this repository.  Nothing from it is copied: the makers
load its files at generation time, with the absent third-party packages stubbed by make_golden.py.
"""
import ast
import copy
import os
import sys
import typing

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("HYDRAGNN_REF", os.path.join(os.path.dirname(ROOT), "reference"))
for _p in (ROOT, os.path.dirname(HERE), HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

HEAD_GRAPH = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                               "dim_headlayers": [10, 7]}}]}
HEAD_NODE = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 6], "type": "mlp"}}]}


# ---- batches and targets ------------------------------------------------------------------------------------------------------
def pna_batch(gen, sizes, input_dim):
    """Random directed edges inside every graph: uneven in-degrees, some nodes without incoming edges, duplicate pairs allowed."""
    from hydragnn_b200.data import Batch, Data
    samples = []
    for n in sizes:
        ne = int(torch.randint(n, 3 * n, (1,), generator=gen))
        src = torch.randint(0, n, (ne,), generator=gen)
        dst = torch.randint(0, max(n - 2, 1), (ne,), generator=gen)          # the last two nodes receive nothing
        keep = src != dst
        ei = torch.stack([src[keep], dst[keep]]).long()
        samples.append(Data(x=torch.randint(1, 9, (n, input_dim), generator=gen).float(), pos=torch.rand(n, 3, generator=gen) * 4.0,
                            edge_index=ei, edge_shifts=torch.zeros(ei.shape[1], 3), y=torch.randn(1, 1, generator=gen)))
    return Batch.from_data_list(samples)


def add_edge_and_pe(b, gen, ekind, edge_dim, use_gps):
    """The edge attribute of a case (``"length"``: the edge lengths; ``"random"``: ``edge_dim`` normal features) and, under GPS,
    the positional encodings the reference's data loader adds."""
    if ekind == "length":
        b.edge_attr = (b.pos[b.edge_index[1]] - b.pos[b.edge_index[0]]).norm(dim=1, keepdim=True)
    elif ekind == "random":
        b.edge_attr = torch.randn(b.edge_index.shape[1], edge_dim, generator=gen)
    if use_gps:
        b.pe = torch.randn(b.x.shape[0], 4, generator=gen)
        b.rel_pe = (b.pe[b.edge_index[0]] - b.pe[b.edge_index[1]]).abs()
    return b


def degree_histogram(b):
    deg = torch.bincount(b.edge_index[1], minlength=b.x.shape[0])
    return torch.bincount(deg).tolist()


def targets(b, kinds, gen):
    """(value, head_index) in the layout Base.loss reads: one flat vector, one index tensor per head."""
    g, n = int(b.batch.max()) + 1, b.x.shape[0]
    vals, idx, off = [], [], 0
    for k in kinds:
        rows = g if k == "graph" else n
        vals.append(torch.randn(rows, generator=gen))
        idx.append(torch.arange(off, off + rows))
        off += rows
    return torch.cat(vals), idx


def t2d(batch):
    return {k: v for k, v in batch.items() if torch.is_tensor(v)}


# ---- one model case -------------------------------------------------------------------------------------------------------------
def record_case(m, b, value, head_index, cfg):
    """The reference stack ``m`` on batch ``b``: its seeded state dict, the eval-mode predictions, and one train-mode step on
    (``value``, ``head_index``) with batch statistics and every dropout off (``nn.Dropout``, GPSConv's and GATv2Conv's own):
    predictions, the reference's own loss, every parameter gradient (None where the reference's is None) and the BatchNorm
    running statistics afterwards."""
    state = {k: v.clone() for k, v in m.state_dict().items()}
    m.eval()
    pred_eval = [p.detach() for p in m(b)]
    m.train()
    for sub in m.modules():
        if isinstance(sub, torch.nn.Dropout):
            sub.p = 0.0
        if type(sub).__name__ in ("GPSConv", "GATv2Conv"):
            sub.dropout = 0.0
    pred = m(b)
    loss, _ = m.loss(pred, value, head_index)
    grads = torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)
    return {"state": state, "inputs": t2d(b), "pred_eval": pred_eval, "pred_train": [p.detach() for p in pred], "value": value,
            "head_index": head_index, "loss": loss.detach(), "str": str(m),
            "state_after": {k: v.clone() for k, v in m.state_dict().items() if "running" in k or "num_batches" in k},
            "grads": {n: (g.detach() if g is not None else None) for (n, _), g in zip(m.named_parameters(), grads)}, "cfg": cfg}


def refusal(fn, **extra):
    """None when ``fn()`` returns; otherwise what the reference raised, ``{"type", "msg"}``, followed by ``extra``."""
    try:
        fn()
    except Exception as e:                                           # noqa: BLE001 -- the reference's own exception is the datum
        return {"type": type(e).__name__, "msg": str(e), **extra}
    return None


# ---- the drop-in dispatch -------------------------------------------------------------------------------------------------------
DISPATCH = '''
import os
if os.getenv("HYDRAGNN_ENGINE", "").lower() == "b200":
    import hydragnn_b200
    if mpnn_type in hydragnn_b200.create.SUPPORTED and global_attn_type in (None, "multihead"):
        return hydragnn_b200.create_model(**{k: v for k, v in locals().items()
                                             if k in hydragnn_b200.create_model.__code__.co_varnames})
'''
# what train / validate / test read through ``model.module`` (train_validate_test.py:225-242,498,731,736,1006-1018)
ATTRS = ("num_heads", "head_dims", "head_type", "loss_weights", "var_output", "graph_pooling")


def reference_create():
    """(create_model_config, create_model) of the reference (hydragnn/models/create.py:41-108,112-766) with the INTEGRATION.md
    dispatch prepended to ``create_model``, on the stubs of make_golden.py.  This re-installs those stubs: a maker installs its
    stack's own after it and hands the stack class to ``create_model_config.__globals__``."""
    import make_golden as mg
    egcl, painn = mg.install_stubs()
    tree = ast.parse(open(REF + "/hydragnn/models/create.py").read())
    fns = {n.name: n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in ("create_model_config", "create_model")}
    assert set(fns) == {"create_model_config", "create_model"}
    fns["create_model"].body = ast.parse(DISPATCH).body + fns["create_model"].body       # the maintainer's patch
    glb = {"torch": torch, "os": os}
    mg._extract(REF + "/hydragnn/utils/model/model.py", ["update_multibranch_heads"], glb)

    class Timer:
        def __init__(self, *_): pass
        def start(self): pass
        def stop(self): pass

    def resolve_precision(p):                         # hydragnn/train/train_validate_test.py:43-63, fp32 / bf16 branch
        return ("fp32", torch.float32, None) if str(p).lower() in ("fp32", "float32") else ("bf16", torch.float32, torch.bfloat16)

    glb.update(Timer=Timer, resolve_precision=resolve_precision, get_device=lambda *a, **k: torch.device("cpu"),
               EGCLStack=egcl.EGCLStack, PAINNStack=painn.PAINNStack, Base=sys.modules["hydragnn.models.Base"].Base,
               List=typing.List, Union=typing.Union, Data=object, torch_scatter=sys.modules["torch_scatter"])
    for name in ("GINStack", "PNAStack", "PNAPlusStack", "GATStack", "MFCStack", "CGCNNStack", "SAGEStack", "SCFStack", "DIMEStack",
                 "PNAEqStack", "MACEStack", "MultiTaskModelMP"):
        glb.setdefault(name, None)
    for n in ("create_model_config", "create_model"):
        exec(compile(ast.Module(body=[fns[n]], type_ignores=[]), REF + "/hydragnn/models/create.py", "exec"), glb)
    return glb["create_model_config"], glb["create_model"]


GPS = dict(pe_dim=6, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=4)


def dropin_config(mpnn_type, output_type, **arch):
    """test_cpu_dropin's configuration of a graph- or node-head ``mpnn_type`` model with ``arch`` set: one head of
    ``output_type``, a node head with layers [50, 25]."""
    from test_cpu_dropin import _config
    cfg = _config(mpnn_type, False)
    cfg["Architecture"].update(output_type=[output_type], **arch)
    if output_type == "node":
        cfg["Architecture"]["output_heads"] = {"node": [{"type": "branch-0", "architecture": {"num_headlayers": 2,
                                                                                              "dim_headlayers": [50, 25],
                                                                                              "type": "mlp"}}]}
    return cfg


def record_dropin(create_model_config, cfg):
    """``create_model_config(cfg)`` of the reference with ``HYDRAGNN_ENGINE`` unset (the reference's own model) and set (the
    engine's, through the dispatch): the config, the keyword arguments the dispatch hands to ``hydragnn_b200.create_model``, and
    what the reference's model shows the training loop -- state dict, ``ATTRS`` and ``str`` of the stack (inside the MLIP wrapper
    where there is one).  Returns (record, the reference's model)."""
    import hydragnn_b200 as hb
    os.environ.pop("HYDRAGNN_ENGINE", None)
    ref = create_model_config(cfg, verbosity=0, use_gpu=False)                    # the reference's own stack
    inner = getattr(ref, "model", ref)
    assert not type(inner).__module__.startswith("hydragnn_b200")
    seen = {}
    real = hb.create_model

    class Spy:                                  # records what the dispatch passes; it filters by create_model's argument names
        __code__ = real.__code__

        def __call__(self, **kw):
            seen.update(kw)
            return real(**kw)

    hb.create_model = Spy()
    os.environ["HYDRAGNN_ENGINE"] = "b200"
    try:
        eng = create_model_config(cfg, verbosity=0, use_gpu=False)                # SAME call, engine behind it
    finally:
        hb.create_model = real
        os.environ.pop("HYDRAGNN_ENGINE", None)
    assert seen and type(getattr(eng, "model", eng)).__module__.startswith("hydragnn_b200")
    return {"config": cfg, "kwargs": seen, "state_dict": {k: v.clone() for k, v in ref.state_dict().items()},
            "attrs": {a: getattr(ref, a) for a in ATTRS}, "repr": str(inner)}, ref


# ---- saving ------------------------------------------------------------------------------------------------------------------
def _own(x, memo):
    if torch.is_tensor(x):
        key = (x.untyped_storage().data_ptr(), x.storage_offset(), tuple(x.shape), tuple(x.stride()), x.dtype)
        if key not in memo:
            memo[key] = x.detach().clone()
        return memo[key]
    if isinstance(x, dict):
        y = copy.copy(x)                                 # same type and attributes: a state dict keeps its _metadata
        y.update((k, _own(v, memo)) for k, v in x.items())
        return y
    if isinstance(x, (list, tuple)):
        return type(x)(_own(v, memo) for v in x)
    return x


def save(obj, path, compact=True):
    """``torch.save(obj, path)``, by default with every tensor first copied into its own compact storage (views of one storage
    stay one tensor).  torch.save writes whole storages, so without the copy a file holds whatever else shares a tensor's
    storage, uninitialised bytes included.  ``compact=False`` writes ``obj`` as it is, for the goldens first written that way
    whose tensors already fill their storages: copying would change their bytes, not their content."""
    torch.save(_own(obj, {}) if compact else obj, path)
    print("written", path)
