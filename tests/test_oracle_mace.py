"""CPU tests of the MACE oracle (oracle/e3.py, oracle/mace.py).  e3nn cannot be installed here and the reference holds no
value pins for MACE (SURVEY.md 8c: "parity unpinned"), so the restatement is checked through the properties the
reference's own MACE tests use (tests/test_forces_equivariant.py:566-710: rotation / translation invariance of the
energy, equivariance of the forces) plus the algebraic identities of the Clebsch-Gordan tensors."""
import math

import pytest
import torch

import hydragnn_b200 as hb
from oracle import e3, mace
from stack_support import MACE_KW, mace_batch, random_rotation

def test_irreps_bookkeeping():
    ir = e3.Irreps("64x0e + 64x1o")
    assert ir.dim == 256 and ir.num_irreps == 128 and ir.count("0e") == 64 and ir.lmax == 1 and "1o" in ir and "1e" not in ir
    sh = e3.Irreps.spherical_harmonics(2)
    assert repr(sh) == "1x0e+1x1o+1x2e"
    assert repr((sh * 4).sort()[0].simplify()) == "4x0e+4x1o+4x2e"
    assert e3.Irrep("1o") < e3.Irrep("1e") < e3.Irrep("2e")            # tuple ordering (l, p)
    assert [repr(x) for x in e3.Irrep("1o") * e3.Irrep("2e")] == ["1o", "2o", "3o"]
    assert e3.create_irreps_string(8, 1) == "8x0e + 8x1o"
    irreps_mid, ins = mace.tp_out_irreps_with_instructions(e3.Irreps("4x0e+4x1o"), sh, e3.Irreps("4x0e+4x1o+4x2e"))
    assert repr(irreps_mid.simplify()) == "8x0e+12x1o+8x2e" and len(ins) == 7 and [i[2] for i in ins] == list(range(7))


@pytest.mark.parametrize("l1,l2,l3", [(1, 1, 0), (1, 1, 1), (1, 1, 2), (1, 2, 3), (2, 2, 2), (2, 2, 4), (1, 2, 2), (2, 1, 1), (3, 2, 1)])
def test_wigner_3j_identities(l1, l2, l3):
    c = e3.wigner_3j(l1, l2, l3)
    assert abs(float(c.norm()) - 1) < 1e-12
    # orthogonality: sum_{m1 m2} C[m1 m2 m3] C[m1 m2 m3'] = delta / (2 l3 + 1)
    g = torch.einsum("ijk,ijl->kl", c, c)
    assert torch.allclose(g, torch.eye(2 * l3 + 1, dtype=torch.float64) / (2 * l3 + 1), atol=1e-12)
    # invariance under rotations, with D^l read off the spherical harmonics themselves
    gen = torch.Generator().manual_seed(5)
    rot = random_rotation(gen)
    pts = torch.randn(64, 3, generator=gen, dtype=torch.float64)

    def d_matrix(l):
        y0 = e3.spherical_harmonics(l, pts)[:, l * l:(l + 1) ** 2]
        y1 = e3.spherical_harmonics(l, pts @ rot.T)[:, l * l:(l + 1) ** 2]
        return torch.linalg.lstsq(y0, y1).solution.T                  # Y(R x) = D Y(x)
    d1, d2, d3 = d_matrix(l1), d_matrix(l2), d_matrix(l3)
    assert torch.allclose(d1 @ d1.T, torch.eye(2 * l1 + 1, dtype=torch.float64), atol=1e-10)
    assert torch.allclose(torch.einsum("ia,jb,kc,abc->ijk", d1, d2, d3, c), c, atol=1e-10)


def test_wigner_3j_low_orders_are_delta_and_epsilon():
    assert torch.allclose(e3.wigner_3j(1, 1, 0).squeeze() * math.sqrt(3), torch.eye(3, dtype=torch.float64), atol=1e-12)
    eps = torch.zeros(3, 3, 3, dtype=torch.float64)
    for i, j, k in [(0, 1, 2), (1, 2, 0), (2, 0, 1)]:
        eps[i, j, k], eps[i, k, j] = 1.0, -1.0
    assert torch.allclose(e3.wigner_3j(1, 1, 1) * math.sqrt(6), eps, atol=1e-12)


def test_spherical_harmonics_match_published_polynomials():
    """The closed forms e3nn documents for l <= 3 ('norm' normalisation, y is the polar axis)."""
    gen = torch.Generator().manual_seed(3)
    v = torch.nn.functional.normalize(torch.randn(50, 3, generator=gen, dtype=torch.float64), dim=-1)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    s3, x2z2 = math.sqrt(3), x * x + z * z
    sh20, sh24 = s3 * x * z, s3 / 2 * (z * z - x * x)
    ref = torch.stack([torch.ones_like(x), x, y, z, sh20, s3 * x * y, y * y - 0.5 * x2z2, s3 * y * z, sh24,
                       math.sqrt(5 / 6) * (sh20 * z + sh24 * x), math.sqrt(5) * sh20 * y, math.sqrt(3 / 8) * (4 * y * y - x2z2) * x,
                       0.5 * y * (2 * y * y - 3 * x2z2), math.sqrt(3 / 8) * z * (4 * y * y - x2z2), math.sqrt(5) * sh24 * y,
                       math.sqrt(5 / 6) * (sh24 * z - sh20 * x)], dim=1)
    assert torch.allclose(e3.spherical_harmonics(3, v * 2.5, normalization="norm"), ref, atol=1e-12)
    comp = e3.spherical_harmonics(2, v, normalization="component")
    assert torch.allclose(comp[:, 4:9].pow(2).sum(1), torch.full((50,), 5.0, dtype=torch.float64), atol=1e-12)
    assert torch.equal(e3.spherical_harmonics(2, torch.zeros(1, 3))[0, 1:], torch.zeros(8))   # zero vector: only l = 0 survives


def test_linear_and_tensor_product_normalisation():
    torch.manual_seed(0)
    lin = e3.Linear("16x0e+16x1o", "8x0e+8x1o")
    assert lin.weight.shape == (2 * 16 * 8,)
    x = torch.randn(4000, 64)
    y = lin(x)
    assert abs(float(y.var()) - 1) < 0.35                                # unit variance in -> unit variance out
    sh = e3.Irreps.spherical_harmonics(2)
    mid, ins = mace.tp_out_irreps_with_instructions(e3.Irreps("8x0e"), sh, e3.Irreps("8x0e+8x1o+8x2e"))
    tp = e3.TensorProductUVU("8x0e", sh, mid, ins)
    assert tp.weight_numel == 24
    v = torch.randn(4000, 3)
    out = tp(torch.randn(4000, 8), e3.spherical_harmonics(2, v), torch.randn(4000, 24))
    assert out.shape == (4000, 8 * 9) and abs(float(out.pow(2).mean()) - 1) < 0.35
    net = e3.FullyConnectedNet([8, 16, 16, 4], torch.nn.functional.silu)
    assert [k for k, _ in net.named_parameters()] == ["layer0.weight", "layer1.weight", "layer2.weight"]
    assert abs(e3.normalize2mom_const(torch.nn.functional.silu) - 1.679) < 2e-3
    assert abs(float(net(torch.randn(4000, 8)).pow(2).mean()) - 1) < 0.5


def test_u_matrices_shapes_and_symmetry():
    coupling = e3.Irreps("1x0e+1x1o+1x2e")
    assert mace.u_matrix_real(coupling, "0e", 1).shape == (9, 1)
    assert mace.u_matrix_real(coupling, "0e", 2).shape == (9, 9, 3)
    assert mace.u_matrix_real(coupling, "1o", 2).shape == (3, 9, 9, 4)
    u3 = mace.u_matrix_real(coupling, "0e", 3)
    assert u3.shape[:3] == (9, 9, 9)
    # every basis element is an invariant: contracting with Y (x) Y gives a rotation-invariant scalar
    gen = torch.Generator().manual_seed(2)
    pts = torch.randn(8, 3, generator=gen, dtype=torch.float64)
    rot = random_rotation(gen)
    y0, y1 = e3.spherical_harmonics(2, pts), e3.spherical_harmonics(2, pts @ rot.T)
    u2 = mace.u_matrix_real(coupling, "0e", 2)
    assert torch.allclose(torch.einsum("ijk,ni,nj->nk", u2, y0, y0), torch.einsum("ijk,ni,nj->nk", u2, y1, y1), atol=1e-10)


def test_mace_oracle_invariances_and_state_dict_layout():
    torch.manual_seed(0)
    m = mace.MACEOracle(**MACE_KW).double()
    keys = list(m.state_dict().keys())
    assert keys[:3] == ["atomic_numbers", "r_max", "num_interactions"]
    assert "graph_convs.0.module_1.conv_tp_weights.layer3.weight" in keys and "graph_convs.1.module_2.symmetric_contractions.contractions.0.weights_max" in keys
    assert m.state_dict()["graph_convs.1.module_1.conv_tp_weights.layer3.weight"].shape == (8, 7 * 8)
    assert "graph_convs.1.module_2.symmetric_contractions.contractions.1.weights_max" not in keys   # last layer: scalars only
    gen = torch.Generator().manual_seed(1)
    d = mace_batch(gen)
    out = m(d)
    assert out[0].shape == (2, 1) and out[1].shape == (16, 3)
    rot = random_rotation(gen)
    d2 = hb.Batch(x=d.x, pos=d.pos @ rot.T + torch.tensor([1.0, -2.0, 0.5], dtype=torch.float64), edge_index=d.edge_index, batch=d.batch)
    d2._num_graphs = 2
    out2 = m(d2)
    assert float((out[0] - out2[0]).abs().max()) < 1e-12 and float((out[1] - out2[1]).abs().max()) < 1e-12

    def energy(p):
        dd = hb.Batch(x=d.x, pos=p, edge_index=d.edge_index, batch=d.batch)
        dd._num_graphs = 2
        o = m(dd)
        return o[0].sum() + o[1].pow(2).sum()
    p1 = d.pos.clone().requires_grad_(True)
    f1, = torch.autograd.grad(energy(p1), p1)
    p2 = (d.pos @ rot.T).clone().requires_grad_(True)
    f2, = torch.autograd.grad(energy(p2), p2)
    assert float(f1.abs().max()) > 1e-4 and float((f1 @ rot.T - f2).abs().max()) < 1e-4 * float(f1.abs().max())   # test_forces_equivariant.py:476
    perm = torch.cat([torch.randperm(7, generator=gen), 7 + torch.randperm(9, generator=gen)])
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(16)
    d3 = hb.Batch(x=d.x[perm], pos=d.pos[perm], edge_index=inv[d.edge_index], batch=d.batch)
    d3._num_graphs = 2
    o3 = m(d3)
    assert float((o3[0] - out[0]).abs().max()) < 1e-12 and float((o3[1] - out[1][perm]).abs().max()) < 1e-12


def test_mace_oracle_matches_the_reference_own_code_golden(golden_dir):
    """models_mace.pt: the reference's MACEStack / blocks / symmetric_contraction / cg / irreps_tools executed with e3nn
    stubbed by oracle/e3.py (tests/golden/make_golden.py).  Same seed -> same keys and initial values; same inputs -> same
    outputs, d(objective)/d(pos) and parameter gradients."""
    g = torch.load(golden_dir + "/models_mace.pt")
    for name, c in g.items():
        torch.manual_seed(0)
        m = mace.MACEOracle(**dict(MACE_KW, **c["cfg"]))
        sd = m.state_dict()
        assert list(sd.keys()) == list(c["state"].keys()), name
        for k, v in sd.items():
            assert torch.equal(v, c["state"][k]), (name, k)
        m.eval()
        d = hb.Batch(**{k: v.clone() for k, v in c["inputs"].items()})
        d._num_graphs = 3
        d.pos.requires_grad_(True)
        pred = m(d)
        for p, q in zip(pred, c["pred"]):
            torch.testing.assert_close(p, q, rtol=1e-5, atol=1e-6)
        obj = pred[0].sum() + pred[1].pow(2).sum()
        f, = torch.autograd.grad(obj, d.pos, retain_graph=True)
        torch.testing.assert_close(f, c["dobj_dpos"], rtol=1e-4, atol=1e-7)
        grads = torch.autograd.grad(obj, list(m.parameters()), allow_unused=True)
        for (n, _), gr in zip(m.named_parameters(), grads):
            ref = c["grads"][n]
            assert (gr is None) == (ref is None), (name, n)
            if gr is not None:
                torch.testing.assert_close(gr, ref, rtol=1e-4, atol=1e-6 * max(1.0, float(ref.abs().max())))
    with pytest.raises(AssertionError, match="num_nodes"):
        mace.MACEOracle(**dict(MACE_KW, num_nodes=None))


def test_clebsch_gordan_and_harmonics_against_sympy():
    """Independent of e3nn and of this repo: (i) the SU(2) Clebsch-Gordan coefficients behind the real Wigner 3j equal sympy's
    for every j <= 3; (ii) the restated real harmonics ('integral' normalisation) equal the standard real spherical harmonics
    Z_lm of sympy, evaluated with e3nn's axis convention (polar axis = y: (X, Y, Z)_std = (z, x, y)), up to the fixed sign
    pattern sign(m) = -1 for m < 0, (-1)^m for m > 0 (sympy carries the Condon-Shortley phase, e3nn's basis does not)."""
    sympy = pytest.importorskip("sympy")
    from sympy.physics.quantum.cg import CG
    for j1 in range(4):
        for j2 in range(4):
            for j3 in range(abs(j1 - j2), j1 + j2 + 1):
                for m1 in range(-j1, j1 + 1):
                    for m2 in range(-j2, j2 + 1):
                        if abs(m1 + m2) <= j3:
                            ref = float(CG(j1, m1, j2, m2, j3, m1 + m2).doit())
                            assert abs(ref - e3._su2_cg_coeff(j1, m1, j2, m2, j3, m1 + m2)) < 1e-12, (j1, m1, j2, m2, j3)
    th, ph = sympy.symbols("theta phi", real=True)
    gen = torch.Generator().manual_seed(0)
    v = torch.nn.functional.normalize(torch.randn(4, 3, generator=gen, dtype=torch.float64), dim=-1)
    y = e3.spherical_harmonics(3, v, normalization="integral")
    for l in range(4):
        for m in range(-l, l + 1):
            expr = sympy.Znm(l, m, th, ph).expand(func=True)
            sign = 1.0 if m == 0 else (-1.0 if m < 0 else (-1.0) ** m)
            for row, (x, yy, z) in enumerate(v.tolist()):
                ref = float(sympy.re(expr.evalf(subs={th: math.acos(yy), ph: math.atan2(x, z)})))
                assert abs(float(y[row, l * l + l + m]) - sign * ref) < 1e-12, (l, m)
