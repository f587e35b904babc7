"""Covalent radii in angstrom by atomic number, the table of ``ase.data.covalent_radii`` that MACE's distance transforms read
(hydragnn/utils/model/mace_utils/modules/radial.py:151-245).

Values: B. Cordero et al., "Covalent radii revisited", Dalton Trans. 2008, 2832-2838, as ase tabulates them: carbon is the
sp3 value, Mn, Fe and Co the low-spin values.  Index 0 (ase's dummy element "X") and Z = 97..118, which the paper does not
cover, hold ase's ``missing = 0.2``.

This is the package's only copy: the engine's MACE buffers, the fp64 oracle and the golden makers all read ``COVALENT_RADII``.
"""
import torch

MISSING = 0.2

_Z1_TO_96 = (
    0.31, 0.28,                                                                                      # H He
    1.28, 0.96, 0.84, 0.76, 0.71, 0.66, 0.57, 0.58,                                                  # Li .. Ne
    1.66, 1.41, 1.21, 1.11, 1.07, 1.05, 1.02, 1.06,                                                  # Na .. Ar
    2.03, 1.76, 1.70, 1.60, 1.53, 1.39, 1.39, 1.32, 1.26, 1.24, 1.32, 1.22, 1.22, 1.20, 1.19, 1.20, 1.20, 1.16,   # K .. Kr
    2.20, 1.95, 1.90, 1.75, 1.64, 1.54, 1.47, 1.46, 1.42, 1.39, 1.45, 1.44, 1.42, 1.39, 1.39, 1.38, 1.39, 1.40,   # Rb .. Xe
    2.44, 2.15,                                                                                      # Cs Ba
    2.07, 2.04, 2.03, 2.01, 1.99, 1.98, 1.98, 1.96, 1.94, 1.92, 1.92, 1.89, 1.90, 1.87, 1.87,      # La .. Lu
    1.75, 1.70, 1.62, 1.51, 1.44, 1.41, 1.36, 1.36, 1.32, 1.45, 1.46, 1.48, 1.40, 1.50, 1.50,      # Hf .. Rn
    2.60, 2.21,                                                                                      # Fr Ra
    2.15, 2.06, 2.00, 1.96, 1.90, 1.87, 1.80, 1.69,                                                  # Ac .. Cm
)

COVALENT_RADII = (MISSING,) + _Z1_TO_96 + (MISSING,) * (118 - 96)        # 119 entries, index = atomic number
assert len(COVALENT_RADII) == 119


def covalent_radii_tensor(dtype=None):
    """The table as the reference registers it: ``torch.tensor(ase.data.covalent_radii, dtype=torch.get_default_dtype())``."""
    return torch.tensor(COVALENT_RADII, dtype=torch.get_default_dtype() if dtype is None else dtype)
