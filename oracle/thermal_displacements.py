"""TEST INFRASTRUCTURE — thermal displacement matrices: the specification of ``chg_thermal_displacements``.

* ``ThermalDisplacementSpecKernels``: ``PhononDosSpecKernels`` (oracle/phonon_dos.py) plus an fp64 torch specification
  of the kernel with the arguments of ``CudaKernels.thermal_displacements``, so that
  ``Phonons(..., device="cpu", kernels=ThermalDisplacementSpecKernels())`` runs ``thermal_displacement_matrices`` on
  the host.
* ``mode_weights``: w(nu, T) = (1 + 2 / expm1(h nu / k T)) / nu for nu >= cutoff, else 0.

Never imported by the product path.
"""
from __future__ import annotations

import torch

from chgnet_b200.phonons import H_OVER_KB_K_PER_THZ
from oracle.phonon_dos import PhononDosSpecKernels

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


class ThermalDisplacementSpecKernels(PhononDosSpecKernels):
    """fp64 specifications of the phonon kernels, the thermal displacement sums included."""

    # (q, mode) pairs per chunk of the specification
    td_chunk_pairs = 1 << 14

    def thermal_displacements(self, freqs, eigvecs, temperatures, cutoff_thz, acc):
        """acc[t, k, c] += sum_{q, mode} mode_weights(nu, T_t) Re(e_k e_k^H)[c], e_k = eigvecs[q, mode, 3k : 3k + 3],
        c in Voigt order (xx, yy, zz, yz, xz, xy)."""
        n_q, n3 = freqs.shape
        n_prim = n3 // 3
        chunk = max(1, self.td_chunk_pairs // max(1, n3))
        total = torch.zeros_like(acc, dtype=torch.float64)
        for s in range(0, n_q, chunk):
            w = mode_weights(freqs[s : s + chunk], temperatures, cutoff_thz)  # [Qc, mode, T]
            e = eigvecs[s : s + chunk].to(torch.complex128).reshape(-1, n3, n_prim, 3)
            outer = (e[..., :, None] * e[..., None, :].conj()).real  # [Qc, mode, k, 3, 3]
            total += torch.einsum("qmt,qmkc->tkc", w, outer[..., VOIGT[0], VOIGT[1]])
        acc += total
