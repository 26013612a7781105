"""TEST INFRASTRUCTURE — two-phonon joint densities of states: ``occupations``, n = 1 / expm1(h nu / k T) (0 at
T = 0), the occupations of the specification of ``chg_joint_dos`` (``PhononSpecKernels``, oracle/phonons.py).

Never imported by the product path.
"""
from __future__ import annotations

import torch

from chgnet_b200.phonons import H_OVER_KB_K_PER_THZ


def occupations(freqs, temperatures):
    """[..., T] Bose-Einstein occupations of ``freqs [...]`` (THz, positive) at ``temperatures [T]`` (K), 0 at T = 0."""
    nu = freqs.to(torch.float64)[..., None]
    t = temperatures.to(torch.float64)
    return torch.where(t > 0, 1.0 / torch.expm1(H_OVER_KB_K_PER_THZ * nu / torch.where(t > 0, t, 1.0)), 0.0)


def __getattr__(name):
    """``JointDosSpecKernels`` stays importable from here: it is ``PhononSpecKernels`` (oracle/phonons.py), which
    holds every phonon specification, imported on first use because oracle/phonons.py imports this module."""
    if name == "JointDosSpecKernels":
        from oracle.phonons import PhononSpecKernels

        return PhononSpecKernels
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
