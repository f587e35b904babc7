"""Generate tests/golden/dropin.pt by running the REFERENCE's own ``create_model_config`` / ``create_model``
(hydragnn/models/create.py:41-108,112-766) with the three-line dispatch of INTEGRATION.md inserted.

Needs a HydraGNN checkout (record.REF); nothing from it is copied: the
two functions are AST-extracted at generation time and exec'd with the absent third-party packages stubbed exactly as
make_golden.py does.  Stored per configuration: the keyword arguments the dispatch hands to ``hydragnn_b200.create_model``, and
what the reference's own model shows to the training loop -- state_dict (seeded with ``torch.manual_seed(0)``, create.py:164),
the attributes train / validate / test read through ``model.module`` (train_validate_test.py:225-242,498,731,736,1006-1018)
and ``str(model)``.  tests/test_cpu_dropin.py checks the engine against it.

    python tests/golden/make_dropin_golden.py
"""
from record import HERE, record_dropin, reference_create, refusal, save
from test_cpu_dropin import _config

# the configurations of tests/test_cpu_dropin.py
CASES = [("EGNN", True), ("PAINN", False), ("EGNN", False)]


def main():
    create_model_config, _ = reference_create()
    out = {}
    for mpnn_type, mlip in CASES:
        rec, ref = record_dropin(create_model_config, _config(mpnn_type, mlip))
        # the reference's own error for an unknown mpnn_type (create.py:584)
        unknown = refusal(lambda: create_model_config(_config("NOPE", False), verbosity=0, use_gpu=False))
        out["%s-%s" % (mpnn_type, mlip)] = {
            "kwargs": rec["kwargs"], "state_dict": rec["state_dict"], "attrs": rec["attrs"],
            "mlip_weights": (ref.energy_weight, ref.energy_peratom_weight, ref.force_weight) if mlip else None,
            "repr": rec["repr"], "unknown_mpnn_type_error": unknown and unknown["type"],
        }
    save(out, HERE + "/dropin.pt", compact=False)


if __name__ == "__main__":
    main()
