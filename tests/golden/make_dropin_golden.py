"""Generate tests/golden/dropin.pt by running the REFERENCE's own ``create_model_config`` / ``create_model``
(hydragnn/models/create.py:41-108,112-766) with the three-line dispatch of INTEGRATION.md inserted.

Needs a HydraGNN checkout (``HYDRAGNN_REF``, default ../reference next to this repository); nothing from it is copied: the
two functions are AST-extracted at generation time and exec'd with the absent third-party packages stubbed exactly as
make_golden.py does.  Stored per configuration: the keyword arguments the dispatch hands to ``hydragnn_b200.create_model``, and
what the reference's own model shows to the training loop -- state_dict (seeded with ``torch.manual_seed(0)``, create.py:164),
the attributes train / validate / test read through ``model.module`` (train_validate_test.py:225-242,498,731,736,1006-1018)
and ``str(model)``.  tests/test_cpu_dropin.py checks the engine against it.

    python tests/golden/make_dropin_golden.py
"""
import ast
import importlib.util
import os
import sys
import typing

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("HYDRAGNN_REF", os.path.join(os.path.dirname(ROOT), "reference"))
sys.path.insert(0, ROOT)

DISPATCH = '''
import os
if os.getenv("HYDRAGNN_ENGINE", "").lower() == "b200":
    import hydragnn_b200
    if mpnn_type in hydragnn_b200.create.SUPPORTED and global_attn_type in (None, "multihead"):
        return hydragnn_b200.create_model(**{k: v for k, v in locals().items()
                                             if k in hydragnn_b200.create_model.__code__.co_varnames})
'''

# the configurations of tests/test_cpu_dropin.py
CASES = [("EGNN", True), ("PAINN", False), ("EGNN", False)]
ATTRS = ("num_heads", "head_dims", "head_type", "loss_weights", "var_output", "graph_pooling")


def _reference_create():
    """(create_model_config, create_model) of the reference with the INTEGRATION.md dispatch prepended to ``create_model``."""
    spec = importlib.util.spec_from_file_location("make_golden", os.path.join(HERE, "make_golden.py"))
    mg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mg)
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


def main():
    import hydragnn_b200 as hb
    from test_cpu_dropin import _config         # noqa: E402  (tests/ is on sys.path below)
    create_model_config, _ = _reference_create()
    out = {}
    for mpnn_type, mlip in CASES:
        cfg = _config(mpnn_type, mlip)
        os.environ.pop("HYDRAGNN_ENGINE", None)
        ref = create_model_config(cfg, verbosity=0, use_gpu=False)                  # the reference's own stack
        assert not type(ref.model if mlip else ref).__module__.startswith("hydragnn_b200")
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
            eng = create_model_config(cfg, verbosity=0, use_gpu=False)              # SAME call, engine behind it
        finally:
            hb.create_model = real
            os.environ.pop("HYDRAGNN_ENGINE", None)
        assert seen and type(eng.model if mlip else eng).__module__.startswith("hydragnn_b200")
        try:                                        # the reference's own error for an unknown mpnn_type (create.py:584)
            create_model_config(_config("NOPE", False), verbosity=0, use_gpu=False)
            unknown_error = None
        except Exception as ex:                     # noqa: BLE001 -- recorded, the test checks it
            unknown_error = type(ex).__name__
        out["%s-%s" % (mpnn_type, mlip)] = {
            "kwargs": seen,
            "state_dict": {k: v.clone() for k, v in ref.state_dict().items()},
            "attrs": {a: getattr(ref, a) for a in ATTRS},
            "mlip_weights": (ref.energy_weight, ref.energy_peratom_weight, ref.force_weight) if mlip else None,
            "repr": str(ref.model if mlip else ref),
            "unknown_mpnn_type_error": unknown_error,
        }
    torch.save(out, os.path.join(HERE, "dropin.pt"))


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    main()
