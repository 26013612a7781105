"""TEST INFRASTRUCTURE — phonon densities of states: ``tetrahedron_weights``, the linear tetrahedron closed forms for
one (tetrahedron, band), vectorised, as the specifications of ``chg_tetrahedron_dos`` and ``chg_joint_dos``
(``PhononSpecKernels``, oracle/phonons.py) evaluate them.

Never imported by the product path.
"""
from __future__ import annotations

import torch


def tetrahedron_weights(e, w):
    """For sorted vertex values ``e [..., 4]`` and frequencies ``w [...]`` (broadcast), per unit tetrahedron volume:
    ``n`` = vol{eps <= w}, ``g`` = dn/dw = int delta(w - eps) and ``wt [..., 4]`` = int delta(w - eps) lambda_i, eps the
    linear interpolant and lambda_i the barycentric coordinates (Bloechl; Lambin and Vigneron).  The cross-section
    eps = w is a triangle for w < e1 or w >= e2, else a quadrilateral, cut by its diagonal into two triangles; wt / g
    is the barycentric centroid of the cross-section."""
    e = e.to(torch.float64)
    w = torch.as_tensor(w, dtype=torch.float64).expand(e.shape[:-1])
    e0, e1, e2, e3 = e.unbind(-1)
    r1, r2, r3 = (w >= e0) & (w < e1), (w >= e1) & (w < e2), (w >= e2) & (w < e3)
    one = torch.ones_like(w)

    def div(a, b, m):  # a / b where m holds, 0 elsewhere (b may vanish outside m)
        return torch.where(m, a / torch.where(m, b, one), 0.0)

    # e0 <= w < e1: triangle on the edges 0-1, 0-2, 0-3
    f10, f20, f30 = div(w - e0, e1 - e0, r1), div(w - e0, e2 - e0, r1), div(w - e0, e3 - e0, r1)
    n1 = f10 * f20 * f30
    g1 = 3 * div(f10 * f20, e3 - e0, r1)
    wt1 = torch.stack([g1 * (3 - f10 - f20 - f30), g1 * f10, g1 * f20, g1 * f30], -1) / 3
    # e1 <= w < e2: quadrilateral P02 P03 P13 P12, f_ij = (w - e_j) / (e_i - e_j)
    x = w - e1
    e10, e20, e30, e21, e31 = e1 - e0, e2 - e0, e3 - e0, e2 - e1, e3 - e1
    n2 = div(e10**2 + 3 * e10 * x + 3 * x**2 - div((e20 + e31) * x**3, e21 * e31, r2), e20 * e30, r2)
    f02, f03, f12, f13 = div(w - e2, e0 - e2, r2), div(w - e3, e0 - e3, r2), div(w - e2, e1 - e2, r2), div(w - e3, e1 - e3, r2)
    f20, f30, f21, f31 = 1 - f02, 1 - f03, 1 - f12, 1 - f13
    g2 = 3 * div(f12 * f20 + f21 * f13, e30, r2)
    gs = 3 * div(f13 * f20, e30, r2)  # area of the triangle P02 P03 P13 (x g)
    gr = g2 - gs  # P02 P13 P12
    wt2 = torch.stack([g2 * f02 + gs * f03, g2 * f13 + gr * f12, g2 * f20 + gr * f21, g2 * f31 + gs * f30], -1) / 3
    # e2 <= w < e3: triangle on the edges 0-3, 1-3, 2-3
    f03b, f13b, f23b = div(e3 - w, e3 - e0, r3), div(e3 - w, e3 - e1, r3), div(e3 - w, e3 - e2, r3)
    n3 = torch.where(r3, 1 - f03b * f13b * f23b, 0.0)
    g3 = 3 * div(f03b * f13b, e3 - e2, r3)
    wt3 = torch.stack([g3 * f03b, g3 * f13b, g3 * f23b, g3 * (3 - f03b - f13b - f23b)], -1) / 3
    n = torch.where(w >= e3, 1.0, n1 + n2 + n3)
    return n, g1 + g2 + g3, wt1 + wt2 + wt3


def __getattr__(name):
    """``PhononDosSpecKernels`` stays importable from here: it is ``PhononSpecKernels`` (oracle/phonons.py), which
    holds every phonon specification, imported on first use because oracle/phonons.py imports this module."""
    if name == "PhononDosSpecKernels":
        from oracle.phonons import PhononSpecKernels

        return PhononSpecKernels
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
