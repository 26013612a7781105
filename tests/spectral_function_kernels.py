"""fp64 torch specification of ``chg_self_energy_spectrum`` with the arguments of ``CudaKernels.self_energy_spectrum``.

``SpectralFunctionSpecKernels`` adds it to ``ThreePhononSpecKernels`` (tests/three_phonon_kernels.py), so that
``Phonons(..., fc3=..., device="cpu", kernels=SpectralFunctionSpecKernels())`` runs ``spectral_function`` on the host.
The weights come from ``vertex_weights``, which evaluates n_band points at a time: the points are passed in slices of
n_band, the last one padded with 0, which lies below the cutoff and so gets no weight.  ``class1_sign=-1`` plants the
bug the tests must catch: it flips g1+ - g1-.  ``axes_reversed`` is ``ThreePhononSpecKernels``'.
"""
from __future__ import annotations

import math

import torch

from chgnet_b200.phonons import H_EV_PER_THZ
from oracle.joint_dos import occupations
from three_phonon_kernels import ThreePhononSpecKernels, _mesh_coords, _mesh_index, vertex_weights


class SpectralFunctionSpecKernels(ThreePhononSpecKernels):
    """``ThreePhononSpecKernels`` with the specification of ``chg_self_energy_spectrum``."""

    def __init__(self, *, class1_sign: float = 1.0, axes_reversed: bool = False):
        super().__init__(axes_reversed=axes_reversed)
        self.class1_sign = class1_sign

    def self_energy_spectrum(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, gamma):
        """gamma[t, l, f] += 18 pi / h^2 sum_{q1, l1, l2} p[q1, l, l1, l2] [(1 + n1 + n2) g2(w_f) + (n1 - n2)
        (g1+ - g1-)(w_f)] with the ``vertex_weights`` at the points w_f = omega[f], n1 = n(freqs[q1, l1]) and
        n2 = n(freqs[target - q1, l2]) the ``occupations`` at temperatures[t]."""
        f64 = torch.float64
        dev = freqs.device
        mesh_t = tuple(int(n) for n in mesh)
        size = torch.tensor(mesh_t, device=dev)
        nu = freqs.to(f64)
        nb, n_f = nu.shape[1], omega.shape[0]
        tc = _mesh_coords(torch.tensor(int(target), device=dev), mesh_t, self.axes_reversed)
        i2 = _mesh_index((tc - _mesh_coords(q1.long(), mesh_t, self.axes_reversed)) % size, mesh_t)
        nu1, nu2 = nu[q1.long()], nu[i2]  # [Q1, nb]
        n1 = occupations(torch.where(nu1 >= cutoff_thz, nu1, 1.0), temperatures)  # [Q1, nb, T]
        n2 = occupations(torch.where(nu2 >= cutoff_thz, nu2, 1.0), temperatures)
        c2 = 1.0 + n1[:, :, None, :] + n2[:, None, :, :]  # [Q1, l1, l2, T]
        c1 = self.class1_sign * (n1[:, :, None, :] - n2[:, None, :, :])
        p = p.to(f64)
        k = 18.0 * math.pi / H_EV_PER_THZ**2
        for s in range(0, n_f, nb):
            pts = torch.zeros(nb, dtype=f64, device=dev)
            here = min(nb, n_f - s)
            pts[:here] = omega[s : s + here].to(f64)
            w = vertex_weights(nu, mesh_t, tetrahedra, target, pts, q1, cutoff_thz, self.ise_chunk_items,
                               self.axes_reversed)
            w = w[:, :here]  # [Q1, point, l1, l2, 3]
            g2 = torch.einsum("qlab,qjab,qabt->tlj", p, w[..., 0], c2)
            g1 = torch.einsum("qlab,qjab,qabt->tlj", p, w[..., 1] - w[..., 2], c1)
            gamma[:, :, s : s + here] += k * (g2 + g1)
