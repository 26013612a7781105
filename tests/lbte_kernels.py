"""fp64 torch specification of ``chg_collision_rows`` with the arguments of ``CudaKernels.collision_rows``.

``LbteSpecKernels`` adds it to ``ThreePhononSpecKernels`` (tests/three_phonon_kernels.py), so that
``Phonons(..., fc3=..., device="cpu", kernels=LbteSpecKernels())`` runs ``thermal_conductivity_lbte`` on the host.
Two switches plant the bugs the tests must catch: ``time_reversal=False`` sends the (b) and (c) terms of DESIGN.md
section 12.8 to the columns q1 and q2 instead of -q1 and -q2, and ``class1_sign=-1`` flips u_q u_c of the class-1
terms.  ``axes_reversed`` is ``ThreePhononSpecKernels``'.
"""
from __future__ import annotations

import math

import torch

from chgnet_b200.phonons import H_EV_PER_THZ, H_OVER_KB_K_PER_THZ
from three_phonon_kernels import ThreePhononSpecKernels, _mesh_coords, _mesh_index, vertex_weights

# 2 pi K, K = 18 pi / h^2: the factor of every term of S (1/ps)
TWO_PI_K = 2.0 * math.pi * (18.0 * math.pi / H_EV_PER_THZ**2)


def inverse_sinh(nu, temperatures, cutoff_thz):
    """[..., T] 1 / sinh(h nu / 2 k T), 0 below ``cutoff_thz`` and at T = 0."""
    t = temperatures.to(torch.float64)
    live = (nu >= cutoff_thz)[..., None] & (t > 0)
    x = 0.5 * H_OVER_KB_K_PER_THZ * torch.where(nu >= cutoff_thz, nu, 1.0)[..., None] / torch.where(t > 0, t, 1.0)
    return torch.where(live, 1.0 / torch.sinh(x), 0.0)


class LbteSpecKernels(ThreePhononSpecKernels):
    """``ThreePhononSpecKernels`` with the specification of ``chg_collision_rows``."""

    def __init__(self, *, time_reversal: bool = True, class1_sign: float = 1.0, axes_reversed: bool = False):
        super().__init__(axes_reversed=axes_reversed)
        self.time_reversal, self.class1_sign = time_reversal, class1_sign

    def collision_rows(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, out):
        """out[:, :, :, q1] = the role sums R_A, R_B, R_C, R_D [4, T, l, q1, b] of the ``vertex_weights`` (g2, g1+,
        g1-) and P = p: A = -2 pi K sum_k P[l, b, k] (g2 + g1-) / s(nu2_k), B = +2 pi K sum_k P[l, b, k] g1+ / s(nu2_k),
        C = -2 pi K sum_k P[l, k, b] (g2 + g1+) / s(nu1_k), D = +2 pi K sum_k P[l, k, b] g1- / s(nu1_k)."""
        f64 = torch.float64
        dev = freqs.device
        mesh_t = tuple(int(n) for n in mesh)
        size = torch.tensor(mesh_t, device=dev)
        nu = freqs.to(f64)
        w = vertex_weights(nu, mesh_t, tetrahedra, target, omega, q1, cutoff_thz, self.ise_chunk_items,
                           self.axes_reversed)
        tc = _mesh_coords(torch.tensor(int(target), device=dev), mesh_t, self.axes_reversed)
        c1 = _mesh_coords(q1.long(), mesh_t, self.axes_reversed)
        i2 = _mesh_index((tc - c1) % size, mesh_t)
        is1 = inverse_sinh(nu[q1.long()], temperatures, cutoff_thz)  # [Q1, nb, T]
        is2 = inverse_sinh(nu[i2], temperatures, cutoff_thz)
        p = p.to(f64)
        g2, gp, gm = w[..., 0], w[..., 1], w[..., 2]
        u = self.class1_sign
        # one temperature at a time, so that a result does not depend on the others in the call
        a = torch.stack([-TWO_PI_K * torch.einsum("qlbk,qk->lqb", p * (g2 + u * gm), x) for x in is2.unbind(-1)])
        b = torch.stack([u * TWO_PI_K * torch.einsum("qlbk,qk->lqb", p * gp, x) for x in is2.unbind(-1)])
        c = torch.stack([-TWO_PI_K * torch.einsum("qlkb,qk->lqb", p * (g2 + u * gp), x) for x in is1.unbind(-1)])
        d = torch.stack([u * TWO_PI_K * torch.einsum("qlkb,qk->lqb", p * gm, x) for x in is1.unbind(-1)])
        # the gather reads R_B at -c and R_D at q + c for column c: without time reversal, vertex q1's R_B lands on
        # column q1 (index -q1) and its R_D on column q2 (index q + q2)
        at_b = q1.long() if self.time_reversal else _mesh_index((-c1) % size, mesh_t)
        at_d = q1.long() if self.time_reversal else _mesh_index((2 * tc - c1) % size, mesh_t)
        out[0][:, :, q1.long()] = a
        out[1][:, :, at_b] = b
        out[2][:, :, q1.long()] = c
        out[3][:, :, at_d] = d
