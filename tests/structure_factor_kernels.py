"""fp64 torch specifications of ``chg_structure_factors`` and ``chg_broadened_spectrum`` with the arguments of
``CudaKernels.structure_factors`` and ``CudaKernels.broadened_spectrum``.

``StructureFactorSpecKernels`` adds them to ``PhononSpecKernels`` (oracle/phonons.py), so that
``Phonons(..., device="cpu", kernels=StructureFactorSpecKernels())`` runs ``dynamic_structure_factor`` and
``powder_spectrum`` on the host.  The occupations are ``oracle.joint_dos.occupations``.
"""
from __future__ import annotations

import math

import torch

from chgnet_b200.phonons import DISPLACEMENT_A2_AMU_THZ
from oracle.joint_dos import occupations
from oracle.phonons import PhononSpecKernels
from oracle.thermal_displacements import VOIGT


class StructureFactorSpecKernels(PhononSpecKernels):
    """``PhononSpecKernels`` with the specifications of the two structure-factor kernels."""

    # rows per chunk of the broadening specification
    sqw_chunk_rows = 1 << 10

    def structure_factors(self, freqs, eigvecs, kcart, gvec, frac, coef, u, temperatures, cutoff_thz, out):
        """out[t, r, m] = (S+, S-) = C (n + 1, n) / nu |F|^2 for nu >= cutoff (else 0), with
        F = sum_k coef_k exp(-K^T U_t,k K / 2) (K . e_k) exp(-2 pi i G . x_k), e_k = eigvecs[r, m, 3k : 3k + 3],
        K = kcart[r], G = gvec[r], x_k = frac[k], U_t,k from the Voigt u[t, k] (W = 0 for u None),
        n = occupations(nu, T_t) and C = ``DISPLACEMENT_A2_AMU_THZ``."""
        f64, c128 = torch.float64, torch.complex128
        n_q, n3 = freqs.shape
        n_prim = n3 // 3
        nu = freqs.to(f64)
        k = kcart.to(f64)
        e = eigvecs.to(c128).reshape(n_q, n3, n_prim, 3)
        ke = torch.einsum("qa,qmka->qmk", k.to(c128), e)
        phase = torch.exp(-2j * math.pi * (gvec.to(f64) @ frac.to(f64).T))  # [Q, k]
        base = ke * (coef.to(f64)[None, :] * phase)[:, None, :]  # [Q, m, k]
        n_t = temperatures.shape[0]
        if u is None:
            dw = torch.ones(n_t, n_q, n_prim, dtype=f64, device=nu.device)
        else:
            u33 = torch.zeros(n_t, n_prim, 3, 3, dtype=f64, device=nu.device)
            u33[..., VOIGT[0], VOIGT[1]] = u.to(f64)
            u33[..., VOIGT[1], VOIGT[0]] = u.to(f64)
            dw = torch.exp(-0.5 * torch.einsum("qa,qb,tkab->tqk", k, k, u33))
        f = torch.einsum("tqk,qmk->tqm", dw.to(c128), base)
        f2 = f.real**2 + f.imag**2
        keep = nu >= cutoff_thz
        safe = torch.where(keep, nu, 1.0)
        n = occupations(safe, temperatures).permute(2, 0, 1)  # [T, Q, m]
        s = torch.where(keep, DISPLACEMENT_A2_AMU_THZ * f2 / safe, 0.0)
        out.copy_(torch.stack([s * (n + 1.0), s * n], -1))

    def broadened_spectrum(self, freqs, weights, row0, group_size, omega, sigma, out):
        """out[t, g] += (1 / group_size) sum over the rows r of group g among [row0, row0 + Q) (r // group_size = g)
        and their modes of S+ g(omega - nu) + S- g(omega + nu), g(x) = exp(-x^2 / 2 sigma^2) / (sigma sqrt(2 pi)) for
        |x| <= 8 sigma, else 0."""
        f64 = torch.float64
        nu, w, om = freqs.to(f64), weights.to(f64), omega.to(f64)
        n_q = nu.shape[0]

        def gauss(x):
            return torch.where(x.abs() <= 8.0 * sigma, torch.exp(-x * x / (2.0 * sigma * sigma)), 0.0) / (
                sigma * math.sqrt(2.0 * math.pi))

        total = torch.zeros_like(out, dtype=f64)
        for s in range(0, n_q, self.sqw_chunk_rows):
            v = nu[s : s + self.sqw_chunk_rows, :, None]  # [Qc, m, 1]
            r = (torch.einsum("tqm,qmf->tqf", w[:, s : s + self.sqw_chunk_rows, :, 0], gauss(om - v))
                 + torch.einsum("tqm,qmf->tqf", w[:, s : s + self.sqw_chunk_rows, :, 1], gauss(om + v)))
            rows = torch.arange(row0 + s, row0 + s + v.shape[0], device=nu.device)
            total.index_add_(1, rows // group_size, r)
        out += total / group_size
