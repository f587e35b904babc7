"""Generate tests/golden/models_mace_transform.pt by running the REFERENCE's own MACEStack with distance_transform "Agnesi" and
"Soft" (mace_utils/modules/radial.py:151-245, blocks.py:141-177, MACEStack.py:171-177, 452-466), on the same stubs as
make_golden.py (e3nn restated by oracle/e3.py, opt_einsum_fx the identity, torch_scatter.scatter index_add_), with the
``ase.data`` stub's covalent radii pointed at hydragnn_b200/covalent_radii.py.  Run where the reference checkout is
(record.REF); the tests never read it.

    python tests/golden/make_mace_transform_golden.py      # writes tests/golden/models_mace_transform.pt, nothing else

Every case records the seeded state dict, the eval-mode outputs, d obj / d pos and the parameter gradients of
obj = pred[0].sum() + pred[1].pow(2).sum(); state dicts and gradients are packed by dtype (``pack``).  The "_mlip" cases (one node head) record instead the reference's own
energy_force_loss (hydragnn/models/create.py, AST-extracted as make_golden.py does): the loss, its tasks, the forces and the
force loss's parameter gradients.  The species cover the missing-radius elements (Z >= 97) and values the reference clamps.
"""
import sys
import types

import numpy as np
import torch

import make_golden as mg
from record import HERE, REF, save, t2d
from hydragnn_b200.covalent_radii import COVALENT_RADII

CONFIGS = {   # name: (distance_transform, radial_type, max_ell, node_max_ell, correlation, num_conv_layers, hidden_dim, mlip)
    "agnesi_bessel": ("Agnesi", "bessel", 2, 1, 2, 2, 4, False),
    "soft_bessel": ("Soft", "bessel", 2, 1, 2, 2, 4, False),
    "soft_chebyshev": ("Soft", "chebyshev", 2, 1, 2, 1, 4, False),
    "agnesi_gaussian_mlip": ("Agnesi", "gaussian", 2, 1, 2, 2, 4, True),
    "soft_gaussian_mlip": ("Soft", "gaussian", 2, 1, 2, 2, 4, True),
}
SPECIES = torch.tensor([1, 6, 7, 8, 26, 29, 79, 96, 97, 100, 118, 0, 130, 1, 6, 8])   # 0 and 130 are clamped to 1 and 118


def pack(tensors):
    """{name: tensor or None} as one flat tensor per dtype plus names, shapes and dtypes: a few hundred small tensors saved one by
    one would make most of the file their per-record overhead.  tests/test_oracle_mace_transform.py's ``unpack`` inverts it."""
    names, shapes, dtypes, flat = [], [], [], {}
    for k, v in tensors.items():
        names.append(k)
        shapes.append(None if v is None else list(v.shape))
        dtypes.append(None if v is None else str(v.dtype).replace("torch.", ""))
        if v is not None:
            flat.setdefault(dtypes[-1], []).append(v.detach().reshape(-1))
    return {"names": names, "shapes": shapes, "dtypes": dtypes, "flat": {k: torch.cat(v) for k, v in flat.items()}}


def main():
    mg.install_stubs()
    mace = mg.install_mace_stubs()
    sys.modules["ase.data"].covalent_radii = np.array(COVALENT_RADII, dtype=np.float64)
    glb = {"torch": torch, "torch_scatter": sys.modules["torch_scatter"]}
    mg._extract(REF + "/hydragnn/models/create.py", ["energy_force_loss"], glb)
    gen = torch.Generator().manual_seed(20261018)
    heads = {"graph": [{"type": "branch-0", "architecture": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                              "dim_headlayers": [10, 6]}}],
             "node": [{"type": "branch-0", "architecture": {"num_headlayers": 2, "dim_headlayers": [12, 12], "type": "mlp"}}]}
    out = {}
    for name, (dtf, radial, max_ell, node_max_ell, corr, layers, hidden, mlip) in CONFIGS.items():
        b = mg.toy_batch(gen, [7, 9, 5], 3.5, input_dim=1)
        b.x = SPECIES[torch.randint(0, len(SPECIES), (b.x.shape[0],), generator=gen)].float()[:, None]
        b.y = torch.randn(b.x.shape[0], 1, generator=gen)
        out_dim, out_type, loss = ([1], ["node"], "mse") if mlip else ([1, 3], ["graph", "node"], "mae")
        torch.manual_seed(0)
        m = mace.MACEStack("node_attributes, equiv_node_feat, inv_node_feat, edge_attributes, edge_features, edge_index",
                           "node_attributes, edge_attributes, edge_features, edge_index", 6.0, radial, dtf, 8, 0,
                           max_ell, node_max_ell, 10.0, 5, corr, 1, hidden, out_dim, 0, "", "", 0, out_type,
                           {"node": heads["node"]} if mlip else heads, "relu", loss, None,
                           loss_weights=[1.0] * len(out_dim), freeze_conv=False, initial_bias=None, num_conv_layers=layers,
                           num_nodes=9, graph_pooling="mean")
        m.eval()
        state = {k: v.clone() for k, v in m.state_dict().items()}
        inp = t2d(b)
        pos0 = b.pos.clone().requires_grad_(True)
        b.pos = pos0
        pred = m(b)
        cfg = dict(distance_transform=dtf, radial_type=radial, max_ell=max_ell, node_max_ell=node_max_ell, correlation=corr,
                   num_conv_layers=layers, hidden_dim=hidden)
        rec = {"state": pack(state), "inputs": inp, "pred": [p.detach() for p in pred], "cfg": cfg}
        if mlip:
            fake = types.SimpleNamespace(num_heads=1, head_type=["node"], model=m, loss_function=m.loss_function,
                                         energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
            tot, tasks = glb["energy_force_loss"](fake, pred, b, create_graph=True)
            energy = sys.modules["torch_scatter"].scatter_add(pred[0], b.batch, dim=0).sum()
            forces = -torch.autograd.grad(energy, pos0, retain_graph=True)[0]
            grads = torch.autograd.grad(tot, list(m.parameters()), allow_unused=True)
            rec.update(loss=tot.detach(), tasks=[t.detach() for t in tasks], forces=forces.detach())
            cfg.update(output_dim=[1], output_type=["node"], task_weights=[1.0], loss_function_type="mse",
                       output_heads={"node": heads["node"][0]["architecture"]})
        else:
            obj = pred[0].sum() + pred[1].pow(2).sum()
            rec["dobj_dpos"] = torch.autograd.grad(obj, pos0, retain_graph=True)[0].detach()
            grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
        rec["grads"] = pack({n: g for (n, _), g in zip(m.named_parameters(), grads)})
        out[name] = rec
    save(out, HERE + "/models_mace_transform.pt")


if __name__ == "__main__":
    main()
