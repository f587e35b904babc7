"""ORACLE (test infrastructure only): fp64 restatement of MACE's distance transforms on top of ``oracle.mace.MACEOracle``.

Follows:
  AgnesiTransform, SoftTransform    hydragnn/utils/model/mace_utils/modules/radial.py:151-245
  RadialEmbeddingBlock              mace_utils/modules/blocks.py:141-177
  wiring                            hydragnn/models/MACEStack.py:171-177, 452-466

``distance_transform`` "Agnesi" or "Soft" registers ``radial_embedding.distance_transform`` between ``bessel_fn`` and
``cutoff_fn`` with the reference's buffers (names, order, dtypes, values), the covalent radii read from
hydragnn_b200/covalent_radii.py (ase's table, the package's one copy).  The cutoff reads the raw edge length d, the basis the
transformed one T(d, r0).  Any other value means no transform, and the model is ``MACEOracle`` unchanged.

Pinned by tests/golden/models_mace_transform.pt, which runs the reference's own files (tests/golden/make_mace_transform_golden.py).
"""
import torch
from torch import nn

from .mace import MACEOracle, RadialEmbedding

KINDS = ("Agnesi", "Soft")


def distance_transform_module(kind):
    """AgnesiTransform / SoftTransform with trainable=False: buffers only, in the reference's order and dtypes."""
    from hydragnn_b200.covalent_radii import covalent_radii_tensor
    m, fp = nn.Module(), torch.get_default_dtype()
    if kind == "Agnesi":
        m.register_buffer("q", torch.tensor(0.9183, dtype=fp))
        m.register_buffer("p", torch.tensor(4.5791, dtype=fp))
        m.register_buffer("a", torch.tensor(1.0805, dtype=fp))
        m.register_buffer("covalent_radii", covalent_radii_tensor(fp))
    elif kind == "Soft":
        m.register_buffer("covalent_radii", covalent_radii_tensor(fp))
        m.register_buffer("a", torch.tensor(0.2))
        m.register_buffer("b", torch.tensor(3.0))
    else:
        raise ValueError("unknown distance transform " + str(kind))
    return m


def transform_of_length(kind, d, rsum, params):
    """T(d) with rsum = R[Z_u] + R[Z_v] (radial.py:187-197 / 234-243), in the dtype of d.  ``params``: (q, p, a) for Agnesi,
    (a, b) for Soft."""
    if kind == "Agnesi":
        q, p, a = params
        r0 = 0.5 * rsum
        return (1 + (a * ((d / r0) ** q) / (1 + (d / r0) ** (q - p)))) ** (-1)
    a, b = params
    r0 = rsum / 4
    return d + (1 / 2) * torch.tanh(-(d / r0) - a * ((d / r0) ** b)) + 1 / 2


class TransformRadialEmbedding(RadialEmbedding):
    """RadialEmbedding with ``distance_transform`` registered between ``bessel_fn`` and ``cutoff_fn`` (blocks.py:154-159).  The
    element index of every node and the edge list are set by ``MACETransformOracle`` before each forward."""

    def __init__(self, r_max, num_bessel, num_polynomial_cutoff, radial_type, kind):
        super().__init__(r_max, num_bessel, num_polynomial_cutoff, radial_type, None)
        self.kind = kind
        cutoff = self._modules.pop("cutoff_fn")
        self.distance_transform = distance_transform_module(kind)
        self.cutoff_fn = cutoff
        self.z = self.edge_index = None

    def transformed(self, d):
        """The transformed length of every edge, d [E, 1]."""
        m = self.distance_transform
        r = m.covalent_radii.to(d.dtype)[self.z + 1].unsqueeze(-1)                   # atomic_numbers[argmax(node_attrs)]
        rsum = r[self.edge_index[0]] + r[self.edge_index[1]]
        params = (m.q, m.p, m.a) if self.kind == "Agnesi" else (m.a, m.b)
        return transform_of_length(self.kind, d, rsum, [v.to(d.dtype) for v in params])

    def forward(self, d):
        """blocks.py:164-177: the cutoff of the raw length d, the basis of T(d)."""
        return self._basis(self.transformed(d)) * self._cutoff(d)

    def _cutoff(self, d):
        """RadialEmbedding's polynomial cutoff (radial.py:110-143)."""
        p, rc = self.cutoff_fn.p.to(d.dtype), self.cutoff_fn.r_max.to(d.dtype)
        env = (1.0 - ((p + 1.0) * (p + 2.0) / 2.0) * torch.pow(d / rc, p) + p * (p + 2.0) * torch.pow(d / rc, p + 1)
               - (p * (p + 1.0) / 2) * torch.pow(d / rc, p + 2))
        return env * (d < rc)

    def _basis(self, t):
        """RadialEmbedding's Bessel / Gaussian / Chebyshev basis (radial.py:18-107)."""
        if self.radial_type == "bessel":
            return self.bessel_fn.prefactor.to(t.dtype) * (torch.sin(self.bessel_fn.bessel_weights.to(t.dtype) * t) / t)
        if self.radial_type == "gaussian":
            return torch.exp(self.coeff * torch.pow(t - self.bessel_fn.gaussian_weights.to(t.dtype), 2))
        return torch.special.chebyshev_polynomial_t(t.repeat(1, self.num_basis), self.bessel_fn.n.to(t.dtype).repeat(len(t), 1))


class MACETransformOracle(MACEOracle):
    """MACEOracle with ``distance_transform`` "Agnesi" / "Soft" (MACEStack.py:171-177, 452-466)."""

    def __init__(self, *args, distance_transform=None, **kwargs):
        super().__init__(*args, **kwargs)
        self.transform = distance_transform if distance_transform in KINDS else None
        if self.transform is not None:
            old = self.radial_embedding                        # same key in _modules: the state-dict position is kept
            p_cut = float(old.cutoff_fn.p)
            self.radial_embedding = TransformRadialEmbedding(old.r_max_f, old.num_basis, p_cut, old.radial_type, self.transform)

    def node_attributes(self, x):
        attrs = super().node_attributes(x)
        if self.transform is not None:
            self.radial_embedding.z = torch.argmax(attrs, dim=1)                      # element index Z - 1
        return attrs

    def forward(self, data):
        if self.transform is not None:
            self.radial_embedding.edge_index = data.edge_index
        return super().forward(data)
