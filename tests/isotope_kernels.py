"""fp64 torch specification of ``chg_isotope_scattering`` with the arguments of ``CudaKernels.isotope_scattering``.

``IsotopeSpecKernels`` adds it to the LBTE and Wigner specifications (tests/lbte_kernels.py, tests/wigner_kernels.py),
so that ``Phonons(..., device="cpu", kernels=IsotopeSpecKernels())`` runs ``isotope_linewidths`` and the three thermal
conductivities with ``mass_variances`` on the host.  ``overlaps`` is a module function so that the tests can use it on
its own.  Two switches plant the bugs the tests must catch: ``conj_target=False`` leaves the target eigenvector
unconjugated, and ``per_component=True`` sums |conj(e) e'|^2 over the Cartesian components instead of squaring the sum.
"""
from __future__ import annotations

import math

import torch

from lbte_kernels import LbteSpecKernels
from oracle.phonon_dos import tetrahedron_weights
from three_phonon_kernels import ThreePhononSpecKernels
from wigner_kernels import WignerSpecKernels


def overlaps(e_target, eigvecs, mass_variances, conj_target=True, per_component=False):
    """O [Q', l', l] = sum_k g_k |sum_a conj(e_ka(l)) e_ka(q', l')|^2 for the target's mode-major eigenvectors
    e_target [l, 3n] and eigvecs [Q', l', 3n]."""
    c128 = torch.complex128
    a = e_target.to(c128)
    a = a.conj() if conj_target else a
    n_prim = a.shape[1] // 3
    x = a.view(-1, n_prim, 3)[None, None] * eigvecs.to(c128).view(*eigvecs.shape[:2], 1, n_prim, 3)  # [Q', l', l, k, 3]
    per_atom = (x.abs() ** 2).sum(-1) if per_component else x.sum(-1).abs() ** 2
    return (per_atom * mass_variances.to(torch.float64)).sum(-1)


class IsotopeSpecKernels(LbteSpecKernels, WignerSpecKernels):
    """The LBTE and Wigner specifications with the specification of ``chg_isotope_scattering``."""

    # tetrahedra per chunk of the isotope specification
    iso_chunk_tets = 1 << 11

    def __init__(self, *, conj_target: bool = True, per_component: bool = False):
        ThreePhononSpecKernels.__init__(self)
        self.time_reversal, self.class1_sign = True, 1.0
        self.same_set_pairs, self.rotation = False, None
        self.conj_target, self.per_component = conj_target, per_component

    def isotope_scattering(self, freqs, mesh, tetrahedra, eigvecs, mass_variances, targets, omega, cutoff_thz, gamma):
        """gamma[t, l] = (pi / 4) w^2 / (6 N) sum over the tetrahedra T of the mesh and the bands l' of sum_v
        wt_v(w) O[q_v, l', l], w = omega[t, l], wt the ``tetrahedron_weights`` of the sorted corner values
        freqs[q_v, l'] and O the ``overlaps`` of target t with vertex modes below ``cutoff_thz`` set to 0; 0 where
        w < ``cutoff_thz``."""
        f64 = torch.float64
        dev = freqs.device
        n1, n2, n3 = (int(n) for n in mesh)
        nu = freqs.to(f64)
        n_q, nb = nu.shape
        i, j, k = torch.meshgrid(*(torch.arange(n, device=dev) for n in (n1, n2, n3)), indexing="ij")
        cell = torch.stack([i.reshape(-1), j.reshape(-1), k.reshape(-1)], 1)
        corners = (cell[:, None, None, :] + tetrahedra.long()[None]) % torch.tensor([n1, n2, n3], device=dev)
        qv = ((corners[..., 0] * n2 + corners[..., 1]) * n3 + corners[..., 2]).reshape(-1, 4)  # [6N, 4]
        e, order = torch.sort(nu[qv].permute(0, 2, 1), dim=-1)  # [6N, l', 4] ascending
        qs = torch.gather(qv[:, None, :].expand(-1, nb, 4), 2, order)  # the corner q of each sorted value
        lp = torch.arange(nb, device=dev)
        for t in range(targets.shape[0]):
            w = omega[t].to(f64)
            o = overlaps(eigvecs[int(targets[t])], eigvecs, mass_variances, self.conj_target, self.per_component)
            o = torch.where((nu >= cutoff_thz)[:, :, None], o, 0.0)  # [N, l', l]
            acc = torch.zeros(nb, dtype=f64, device=dev)
            for s in range(0, e.shape[0], self.iso_chunk_tets):
                ec, qc = e[s : s + self.iso_chunk_tets], qs[s : s + self.iso_chunk_tets]
                wt = tetrahedron_weights(ec[:, :, None, :].expand(-1, -1, nb, -1), w[None, None, :])[2]  # [C, l', l, 4]
                ov = o[qc, lp[None, :, None]]  # [C, l', 4, l]
                acc += torch.einsum("cmlv,cmvl->l", wt, ov)
            gamma[t] = torch.where(w >= cutoff_thz, acc * (math.pi / 4 * w * w / (6.0 * n_q)), 0.0)
