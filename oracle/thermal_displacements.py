"""TEST INFRASTRUCTURE — thermal displacement matrices: the weights of the specification of
``chg_thermal_displacements`` (``PhononSpecKernels``, oracle/phonons.py).

* ``mode_weights``: w(nu, T) = (1 + 2 / expm1(h nu / k T)) / nu for nu >= cutoff, else 0.
* ``VOIGT``: the (row, column) pairs of the Voigt order.

Never imported by the product path.
"""
from __future__ import annotations

import torch

from chgnet_b200.phonons import H_OVER_KB_K_PER_THZ

# Voigt order xx, yy, zz, yz, xz, xy
VOIGT = ([0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1])


def mode_weights(freqs, temperatures, cutoff_thz):
    """[..., T] weights of the frequencies ``freqs [...]`` (THz) at ``temperatures [T]`` (K): (1 + 2 n) / nu with
    1 + 2 n = 1 + 2 / expm1(h nu / k T) (1 at T = 0) for nu >= ``cutoff_thz``, and 0 for the modes left out."""
    nu = freqs.to(torch.float64)[..., None]
    t = temperatures.to(torch.float64)
    keep = nu >= cutoff_thz
    safe = torch.where(keep, nu, 1.0)
    x = H_OVER_KB_K_PER_THZ * safe / torch.where(t > 0, t, 1.0)
    coth = torch.where(t > 0, 1.0 + 2.0 / torch.expm1(x), 1.0)
    return torch.where(keep, coth / safe, 0.0)


def __getattr__(name):
    """``ThermalDisplacementSpecKernels`` stays importable from here: it is ``PhononSpecKernels``
    (oracle/phonons.py), which holds every phonon specification, imported on first use because oracle/phonons.py
    imports this module."""
    if name == "ThermalDisplacementSpecKernels":
        from oracle.phonons import PhononSpecKernels

        return PhononSpecKernels
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
