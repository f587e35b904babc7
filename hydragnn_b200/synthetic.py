"""Synthetic radius-graph workloads of the shapes BASELINE.json names (SURVEY.md 8d, configs C1-C3).

Everything is drawn from ``torch.Generator().manual_seed(seed)`` on the CPU so the oracle, the engine and
every rank see identical inputs.  Positions: atoms uniform in a cube at number density ``rho`` with a minimum
separation (rejection-resampled, vectorised over graphs).  Labels are synthetic (standard normal); there is
no network to fetch QM9 / MD17.
"""
import torch

from .data import Batch, Data

WORKLOADS = {
    # name: atoms/graph, density, species pool (atomic numbers), radius, max_neighbours
    "qm9_painn": dict(n=9, rho=0.10, species=[1, 6, 7, 8, 9], radius=7.0, max_neighbours=5),
    "md17_egnn": dict(n=21, rho=0.08, species=[6] * 9 + [1] * 8 + [8] * 4, radius=7.0, max_neighbours=5, fixed_species=True),
    "lj_egnn": dict(n=27, lattice=3.8, radius=5.0, max_neighbours=5, pbc=True),
    # SURVEY C5 (multibranch GFM shape): graph sizes drawn from {9, 21, 80, 200} with equal probability, rho = 0.06, r = 5,
    # k = 20, positional encodings for GPS, graph energy + node forces heads
    "gfm_pnaeq": dict(sizes=[9, 21, 80, 200], rho=0.06, species=list(range(1, 84)), radius=5.0, max_neighbours=20, pe_dim=6,
                      two_heads=True),
    # the same with 40-atom clusters only (unit tests)
    "gfm_pnaeq_mini": dict(n=40, rho=0.06, species=list(range(1, 84)), radius=5.0, max_neighbours=20, pe_dim=6),
    # SURVEY C4 (open-catalyst-like): n ~ U{60..100} atoms in a periodic cubic cell at 0.05 / A^3, Z ~ U{1..83}, r = 6 A,
    # all neighbours
    "oc20_mace": dict(sizes=list(range(60, 101)), rho=0.05, species=list(range(1, 84)), radius=6.0, max_neighbours=128,
                      pbc_box=True, two_heads=True),
    # the same with exactly 80 atoms per cell (unit tests)
    "oc20_mace_80": dict(n=80, rho=0.05, species=list(range(1, 84)), radius=6.0, max_neighbours=128, pbc_box=True, two_heads=True),
    # PNA on examples/eam (NiNb EAM): periodic 32-atom metal cells at a metallic number density, r = 3 A
    "eam_pna": dict(n=32, rho=0.085, species=[28, 41], radius=3.0, max_neighbours=20, pbc_box=True),
    # PNA on examples/ogb (ogb_gap): molecule-sized graphs of 9 to 30 atoms, k = 20
    "ogb_pna": dict(sizes=list(range(9, 31)), rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20),
    # PNAPlus on examples/LennardJones (LJ.json: periodic cells, r = 5, k = 5) and on the ogb_pna graphs
    "lj_pnaplus": dict(n=27, lattice=3.8, radius=5.0, max_neighbours=5, pbc=True),
    "ogb_pnaplus": dict(sizes=list(range(9, 31)), rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20),
    # GAT on the ogb_pna graphs; the GPS variant adds the positional encodings
    "ogb_gat": dict(sizes=list(range(9, 31)), rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20),
    "ogb_gat_gps": dict(sizes=list(range(9, 31)), rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20, pe_dim=6),
    # SAGE and MFC on the ogb_pna graphs; the GPS variant adds the positional encodings
    "ogb_sage": dict(sizes=list(range(9, 31)), rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20),
    "ogb_mfc": dict(sizes=list(range(9, 31)), rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20),
    "ogb_sage_gps": dict(sizes=list(range(9, 31)), rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20, pe_dim=6),
    # SchNet on examples/qm9 and examples/md17 (GPS: the positional encodings pe, rel_pe = |pe[row] - pe[col]| once the edges
    # exist, see add_rel_pe), and without GPS at the CI widths, building its radius graphs in the layers
    "qm9_schnet": dict(n=9, rho=0.10, species=[1, 6, 7, 8, 9], radius=7.0, max_neighbours=5, pe_dim=2),
    "md17_schnet": dict(n=21, rho=0.08, species=[6] * 9 + [1] * 8 + [8] * 4, radius=7.0, max_neighbours=5, fixed_species=True,
                        pe_dim=6),
    "ci_schnet": dict(n=9, rho=0.10, species=[1, 6, 7, 8, 9], radius=5.0, max_neighbours=20),
    # CGCNN on Materials-Project-like crystals: periodic cells of 8 to 64 atoms, any species, CGCNN's 12-neighbour graphs
    # (r = 8 A); the GPS variant adds the positional encodings
    "mp_cgcnn": dict(sizes=list(range(8, 65)), rho=0.06, species=list(range(1, 84)), radius=8.0, max_neighbours=12, pbc_box=True),
    "mp_cgcnn_gps": dict(sizes=list(range(8, 65)), rho=0.06, species=list(range(1, 84)), radius=8.0, max_neighbours=12,
                         pbc_box=True, pe_dim=6),
    # examples/multidataset_hpo_sc26/gfm_mlip.json: MACE force training conditioned on graph attributes (concat_node), periodic
    # cells of 60 to 100 atoms of any species, r = 5 A, k = 20; graph_attr (two per graph) is attached by the caller
    "gfm_mace": dict(sizes=list(range(60, 101)), rho=0.05, species=list(range(1, 84)), radius=5.0, max_neighbours=20, pbc_box=True),
}

ARCH = {
    # examples/qm9/qm9.json minus GPS, mpnn_type PAINN (SURVEY C2)
    "qm9_painn": dict(mpnn_type="PAINN", input_dim=1, hidden_dim=64, num_conv_layers=2, num_radial=5, radius=7.0,
                      max_neighbours=5, output_dim=[1], output_type=["graph"], task_weights=[1.0],
                      output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                              "dim_headlayers": [50, 25]}},
                      activation_function="relu", loss_function_type="mse", graph_pooling="mean"),
    # examples/md17/md17_mlip.json with the three MLIP weights set to 1 (SURVEY C3)
    "md17_egnn": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=64, num_conv_layers=3, num_radial=5, radius=7.0,
                      max_neighbours=5, output_dim=[1], output_type=["node"], task_weights=[1.0],
                      output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [60, 20], "type": "mlp"}},
                      activation_function="relu", loss_function_type="mse", enable_interatomic_potential=True,
                      energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0),
    # SURVEY C5: PNAEq + GPS (examples/multibranch/multibranch_GFM260.json knobs, GPS knobs of qm9.json); pna_deg is filled in
    # from the batch (degree histogram) by the caller
    "gfm_pnaeq": dict(mpnn_type="PNAEq", input_dim=1, hidden_dim=64, num_conv_layers=3, num_radial=6, radius=5.0, max_neighbours=20,
                      global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=8, pe_dim=6,
                      output_dim=[1, 3], output_type=["graph", "node"], task_weights=[1.0, 1.0],
                      output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 50, "num_headlayers": 2, "dim_headlayers": [50, 25]},
                                    "node": {"num_headlayers": 2, "dim_headlayers": [200, 200], "type": "mlp"}},
                      activation_function="relu", loss_function_type="mae", graph_pooling="mean"),
    # SURVEY C4: MACE knobs of tests/test_forces_equivariant.py:318-327, heads of multidataset/gfm_multitasking.json
    "oc20_mace": dict(mpnn_type="MACE", input_dim=1, hidden_dim=64, num_conv_layers=2, num_radial=8, radius=6.0,
                      max_neighbours=128, max_ell=2, node_max_ell=1, correlation=2, envelope_exponent=5, radial_type="bessel",
                      avg_num_neighbors=45.0, num_nodes=80, output_dim=[1, 3], output_type=["graph", "node"], task_weights=[1.0, 1.0],
                      output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 50, "num_headlayers": 2,
                                              "dim_headlayers": [50, 25]},
                                    "node": {"num_headlayers": 2, "dim_headlayers": [200, 200], "type": "mlp"}},
                      activation_function="relu", loss_function_type="mae", graph_pooling="mean"),
    # examples/LennardJones/LJ.json with mpnn_type EGNN, 2 layers (SURVEY C1)
    "lj_egnn": dict(mpnn_type="EGNN", input_dim=1, hidden_dim=32, num_conv_layers=2, radius=5.0, max_neighbours=5,
                    output_dim=[1], output_type=["node"], task_weights=[1.0],
                    output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [60, 20], "type": "mlp"}},
                    activation_function="relu", loss_function_type="mse", enable_interatomic_potential=True,
                    energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0),
}


# PNA (PNAStack.py) at the widths of examples/eam/NiNb_EAM_*.json and examples/ogb/ogb_gap.json; pna_deg is filled in from the
# batch (in-degree histogram) by the caller, eam_pna reads the edge length as a 1-wide edge attribute
ARCH["eam_pna"] = dict(mpnn_type="PNA", input_dim=1, hidden_dim=50, num_conv_layers=10, edge_dim=1, radius=3.0, max_neighbours=20,
                       output_dim=[1], output_type=["node"], task_weights=[1.0],
                       output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [50, 25], "type": "mlp"}},
                       activation_function="relu", loss_function_type="mse", graph_pooling="mean")
ARCH["ogb_pna"] = dict(mpnn_type="PNA", input_dim=1, hidden_dim=55, num_conv_layers=6, radius=5.0, max_neighbours=20,
                       output_dim=[1], output_type=["graph"], task_weights=[1.0],
                       output_heads={"graph": {"num_sharedlayers": 1, "dim_sharedlayers": 55, "num_headlayers": 2,
                                               "dim_headlayers": [55, 55]}},
                       activation_function="relu", loss_function_type="mse", graph_pooling="mean")
# PNAPlus (PNAPlusStack.py): examples/LennardJones/LJ.json (4 layers at 32, 5 radial functions, envelope 5, MLIP with energy,
# per-atom energy and force losses) and the ogb_pna widths with the same basis; pna_deg is filled in by the caller
ARCH["lj_pnaplus"] = dict(mpnn_type="PNAPlus", input_dim=1, hidden_dim=32, num_conv_layers=4, num_radial=5, envelope_exponent=5,
                          radius=5.0, max_neighbours=5, output_dim=[1], output_type=["node"], task_weights=[1.0],
                          output_heads={"node": {"num_headlayers": 2, "dim_headlayers": [60, 20], "type": "mlp"}},
                          activation_function="relu", loss_function_type="mse", enable_interatomic_potential=True,
                          energy_weight=1.0, energy_peratom_weight=1.0, force_weight=1.0)
ARCH["ogb_pnaplus"] = dict(ARCH["ogb_pna"], mpnn_type="PNAPlus", num_radial=5, envelope_exponent=5)
# GAT (GATStack.py, 6 attention heads as create.py fixes them): the ogb_pna graphs and graph head with the edge length as the one
# edge feature, 3 layers at hidden 64 (the concat layers are 6 x 64 = 384 wide; the reference ships no GAT example, 64 is the
# width of the other GPS workloads); the GPS variant adds 8 attention heads and pe_dim 6
ARCH["ogb_gat"] = dict(ARCH["ogb_pna"], mpnn_type="GAT", hidden_dim=64, num_conv_layers=3, edge_dim=1)
ARCH["ogb_gat_gps"] = dict(ARCH["ogb_gat"], global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=8, pe_dim=6)
# SAGE (SAGEStack.py) and MFC (MFCStack.py, max_degree = max_neighbours = 20: 21 weight groups): the ogb_pna graphs and graph
# head, 3 layers at hidden 64; the GPS variant adds 8 attention heads and pe_dim 6
ARCH["ogb_sage"] = dict(ARCH["ogb_pna"], mpnn_type="SAGE", hidden_dim=64, num_conv_layers=3)
ARCH["ogb_mfc"] = dict(ARCH["ogb_sage"], mpnn_type="MFC")
ARCH["ogb_sage_gps"] = dict(ARCH["ogb_sage"], global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=8, pe_dim=6)
# SchNet (SCFStack.py): examples/qm9/qm9.json exactly, examples/md17/md17.json (6 layers, pe_dim 6), and the in-layer branch at
# the widths of tests/inputs/ci.json (num_filters 126, num_gaussians 50) with hidden 64 and three layers
ARCH["qm9_schnet"] = dict(mpnn_type="SchNet", input_dim=1, hidden_dim=64, num_conv_layers=2, num_gaussians=10, num_filters=8,
                          radius=7.0, max_neighbours=5, global_attn_engine="GPS", global_attn_type="multihead", global_attn_heads=8,
                          pe_dim=2, output_dim=[1], output_type=["graph"], task_weights=[1.0],
                          output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 5, "num_headlayers": 2,
                                                  "dim_headlayers": [50, 25]}},
                          activation_function="relu", loss_function_type="mse", graph_pooling="mean")
ARCH["md17_schnet"] = dict(ARCH["qm9_schnet"], num_conv_layers=6, pe_dim=6)
ARCH["ci_schnet"] = dict(mpnn_type="SchNet", input_dim=1, hidden_dim=64, num_conv_layers=3, num_gaussians=50, num_filters=126,
                         radius=5.0, max_neighbours=20, output_dim=[1], output_type=["graph"], task_weights=[1.0],
                         output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 4, "num_headlayers": 2,
                                                 "dim_headlayers": [10, 10]}},
                         activation_function="relu", loss_function_type="mse", graph_pooling="mean")
ARCH["oc20_mace_80"] = ARCH["oc20_mace"]
ARCH["gfm_mace"] = dict(mpnn_type="MACE", input_dim=1, hidden_dim=128, num_conv_layers=4, num_radial=6, radius=5.0, max_neighbours=20,
                        max_ell=1, node_max_ell=1, envelope_exponent=5, radial_type="bessel", avg_num_neighbors=13.735293601560318,
                        edge_dim=1, output_dim=[1], output_type=["graph"], task_weights=[1.0],
                        output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 50, "num_headlayers": 3,
                                                "dim_headlayers": [128, 128, 128]}},
                        activation_function="relu", loss_function_type="mae", graph_pooling="add",
                        enable_interatomic_potential=True, energy_weight=0.0, energy_peratom_weight=1.0, force_weight=10.0,
                        use_graph_attr_conditioning=True, graph_attr_conditioning_mode="concat_node")
ARCH["gfm_pnaeq_mini"] = dict(ARCH["gfm_pnaeq"], output_dim=[1], output_type=["graph"], task_weights=[1.0], loss_function_type="mse",
                              output_heads={"graph": ARCH["gfm_pnaeq"]["output_heads"]["graph"]})
# CGCNN (CGCNNStack.py): the edge length as the one edge feature, and input_dim = hidden_dim = 1 as update_config makes them
# without GPS, with the graph head widths of tests/inputs/ci.json; with GPS (8 heads, pe_dim 6) at hidden 64
ARCH["mp_cgcnn"] = dict(mpnn_type="CGCNN", input_dim=1, hidden_dim=1, num_conv_layers=3, edge_dim=1, radius=8.0, max_neighbours=12,
                        output_dim=[1], output_type=["graph"], task_weights=[1.0],
                        output_heads={"graph": {"num_sharedlayers": 2, "dim_sharedlayers": 4, "num_headlayers": 2,
                                                "dim_headlayers": [10, 10]}},
                        activation_function="relu", loss_function_type="mse", graph_pooling="mean")
ARCH["mp_cgcnn_gps"] = dict(ARCH["mp_cgcnn"], hidden_dim=64, global_attn_engine="GPS", global_attn_type="multihead",
                            global_attn_heads=8, pe_dim=6)


def _cube_positions(gen, num_graphs, n, box, min_sep, max_iter=200):
    pos = torch.rand(num_graphs, n, 3, generator=gen) * box
    eye = torch.eye(n, dtype=torch.bool)
    for _ in range(max_iter):
        d = torch.cdist(pos, pos)
        close = (d < min_sep) & ~eye
        bad = torch.triu(close, 1).any(dim=1)            # the later atom of every too-close pair
        if not bool(bad.any()):
            break
        pos[bad] = torch.rand(int(bad.sum()), 3, generator=gen) * box
    return pos


def _make_mixed(name, num_graphs, seed):
    """Variable-size graphs (``sizes``): every graph draws its atom count from the list with equal probability; positions are
    generated per size group (vectorised) and laid out in graph order."""
    w = WORKLOADS[name]
    gen = torch.Generator().manual_seed(seed)
    sizes = torch.tensor(w["sizes"])
    ns = sizes[torch.randint(0, len(sizes), (num_graphs,), generator=gen)]
    ptr = torch.zeros(num_graphs + 1, dtype=torch.long)
    ptr[1:] = torch.cumsum(ns, 0)
    n_tot = int(ptr[-1])
    pos = torch.empty(n_tot, 3)
    for n in sorted(set(ns.tolist())):
        gi = torch.nonzero(ns == n).flatten()
        box = (n / w["rho"]) ** (1.0 / 3.0)
        p = _cube_positions(gen, gi.numel(), n, box, 0.9)
        rows = (ptr[gi][:, None] + torch.arange(n)[None, :]).reshape(-1)
        pos[rows] = p.reshape(-1, 3)
    sp = torch.tensor(w["species"], dtype=torch.float32)
    out = Batch()
    out.x = sp[torch.randint(0, len(sp), (n_tot,), generator=gen)].reshape(-1, 1).contiguous()
    out.pos = pos
    out.batch = torch.repeat_interleave(torch.arange(num_graphs), ns)
    out.ptr = ptr
    out._num_graphs = num_graphs
    out.energy = torch.randn(num_graphs, generator=gen)
    out.forces = torch.randn(n_tot, 3, generator=gen)
    y = torch.randn(num_graphs, 1, generator=gen)
    if w.get("pe_dim"):
        out.pe = torch.randn(n_tot, w["pe_dim"], generator=gen)
    if w.get("two_heads"):                                  # y = per graph [energy, forces...] with y_loc offsets
        parts = []
        for g in range(num_graphs):
            parts += [y[g], out.forces[ptr[g]:ptr[g + 1]].reshape(-1)]
        out.y = torch.cat(parts).reshape(-1, 1).contiguous()
        out.y_loc = torch.stack([torch.zeros_like(ns), torch.ones_like(ns), 1 + 3 * ns], dim=1).contiguous()
    else:
        out.y = y
    if w.get("pbc_box"):
        L = (ns.double() / w["rho"]) ** (1.0 / 3.0)
        out.cell = (torch.eye(3, dtype=torch.float64)[None] * L[:, None, None]).float().contiguous()
        out.pbc = torch.ones(num_graphs, 3, dtype=torch.bool)
    return out


def make_samples(name, num_graphs, seed=1234, with_edges=None):
    """List-free construction: returns one ``Batch`` (CPU) with x, pos, batch, ptr, y / energy / forces
    (+ cell, pbc for the periodic LJ workload).  Edges are NOT built here -- that is the radius-graph kernel's
    job (or the oracle's, on the CPU side)."""
    w = WORKLOADS[name]
    if "sizes" in w:
        return _make_mixed(name, num_graphs, seed)
    gen = torch.Generator().manual_seed(seed)
    n = w["n"]
    if "lattice" in w:                                      # 3x3x3 simple cubic, jitter +-0.05 a (LJ_data.py:310-343)
        a = w["lattice"]
        grid = torch.stack(torch.meshgrid(*[torch.arange(3.0)] * 3, indexing="ij"), -1).reshape(-1, 3) * a
        pos = grid[None] + (torch.rand(num_graphs, n, 3, generator=gen) - 0.5) * 0.1 * a
        z = torch.ones(num_graphs, n)
    else:
        box = (n / w["rho"]) ** (1.0 / 3.0)
        pos = _cube_positions(gen, num_graphs, n, box, 0.9)
        sp = torch.tensor(w["species"], dtype=torch.float32)
        if w.get("fixed_species"):
            z = sp[None, :].expand(num_graphs, n).clone()
        else:
            z = sp[torch.randint(0, len(sp), (num_graphs, n), generator=gen)]
    out = Batch()
    out.x = z.reshape(-1, 1).contiguous()
    out.pos = pos.reshape(-1, 3).contiguous()
    out.batch = torch.arange(num_graphs).repeat_interleave(n)
    out.ptr = torch.arange(num_graphs + 1) * n
    out._num_graphs = num_graphs
    out.y = torch.randn(num_graphs, 1, generator=gen)
    out.energy = torch.randn(num_graphs, generator=gen)
    out.forces = torch.randn(num_graphs * n, 3, generator=gen)
    if w.get("pe_dim"):
        out.pe = torch.randn(num_graphs * n, w["pe_dim"], generator=gen)
    if w.get("two_heads"):                                  # y = per graph [energy, forces...] with y_loc offsets
        out.y = torch.cat([out.y, out.forces.reshape(num_graphs, 3 * n)], dim=1).reshape(-1, 1).contiguous()
        out.y_loc = torch.tensor([[0, 1, 1 + 3 * n]]).expand(num_graphs, 3).contiguous()
    if w.get("pbc_box"):
        L = (n / w["rho"]) ** (1.0 / 3.0)
        out.cell = (torch.eye(3) * L)[None].expand(num_graphs, 3, 3).contiguous()
        out.pbc = torch.ones(num_graphs, 3, dtype=torch.bool)
    if w.get("pbc"):
        L = 3 * w["lattice"]
        out.cell = (torch.eye(3) * L)[None].expand(num_graphs, 3, 3).contiguous()
        out.pbc = torch.ones(num_graphs, 3, dtype=torch.bool)
    return out


def add_rel_pe(batch):
    """rel_pe = |pe[row] - pe[col]| on the batch's edges (hydragnn/preprocess/serialized_dataset_loader.py:186-189)."""
    row, col = batch.edge_index
    batch.rel_pe = (batch.pe[row] - batch.pe[col]).abs().contiguous()
    return batch
