"""TEST INFRASTRUCTURE — two-phonon joint densities of states: the specification of ``chg_joint_dos``.

* ``JointDosSpecKernels``: ``ThermalDisplacementSpecKernels`` (oracle/thermal_displacements.py) plus an fp64 torch
  specification of the kernel with the arguments of ``CudaKernels.joint_dos``, so that
  ``Phonons(..., device="cpu", kernels=JointDosSpecKernels())`` runs ``joint_dos`` and ``phase_space`` on the host.
  Unlike the kernel, it evaluates both class-1 terms, d(w + nu1 - nu2) and d(w - nu1 + nu2), separately.
* ``occupations``: n = 1 / expm1(h nu / k T) (0 at T = 0).

Never imported by the product path.
"""
from __future__ import annotations

import torch

from chgnet_b200.phonons import H_OVER_KB_K_PER_THZ
from oracle.phonon_dos import tetrahedron_weights
from oracle.thermal_displacements import ThermalDisplacementSpecKernels


def occupations(freqs, temperatures):
    """[..., T] Bose-Einstein occupations of ``freqs [...]`` (THz, positive) at ``temperatures [T]`` (K), 0 at T = 0."""
    nu = freqs.to(torch.float64)[..., None]
    t = temperatures.to(torch.float64)
    return torch.where(t > 0, 1.0 / torch.expm1(H_OVER_KB_K_PER_THZ * nu / torch.where(t > 0, t, 1.0)), 0.0)


class JointDosSpecKernels(ThermalDisplacementSpecKernels):
    """fp64 specifications of the phonon kernels, the joint densities of states included."""

    # (tetrahedron, band pair) items per chunk of the specification
    jdos_chunk_items = 1 << 17

    def joint_dos(self, freqs, mesh, tetrahedra, targets, omega, temperatures, cutoff_thz, out):
        """out [Q, 1 + T, 2, F]: ``joint_dos_terms`` with the two class-1 terms added."""
        terms = self.joint_dos_terms(freqs, mesh, tetrahedra, targets, omega, temperatures, cutoff_thz)
        out.copy_(torch.stack([terms[:, :, 0] + terms[:, :, 1], terms[:, :, 2]], 2))

    def joint_dos_terms(self, freqs, mesh, tetrahedra, targets, omega, temperatures, cutoff_thz):
        """[Q, 1 + T, 3, F]: the three terms below at the frequency points omega[q] of each target, slot 0 with
        c_i = 1 (D2) and slot 1 + t with the occupation factors at temperatures[t] (N2).  Each term is the sum over
        every (cell, tetrahedron T, l1, l2) of sum_i wt_T,i(w) m_i c_i, each tetrahedron weighted 1 / (6 N), with the
        corner values and factors

            d(w + nu1 - nu2): f_i = nu2 - nu1, c_i = 1 | n1 - n2           (class 1)
            d(w - nu1 + nu2): f_i = nu1 - nu2, c_i = 1 | -(n1 - n2)        (class 1)
            d(w - nu1 - nu2): f_i = nu1 + nu2, c_i = 1 | n1 + n2 + 1       (class 2)

        nu1 = freqs[q1_i, l1], nu2 = freqs[q2_i, l2], q1_i the corners of T and q2_i = q - q1_i on the mesh, and
        m_i = 0 where nu1 or nu2 is below ``cutoff_thz``.  Only the points inside [f_0, f_3) of an item are
        evaluated."""
        f64 = torch.float64
        dev = freqs.device
        n1, n2, n3 = (int(n) for n in mesh)
        n_q, n_band = freqs.shape
        nu = freqs.to(f64)
        temps = torch.zeros(0, dtype=f64, device=dev) if temperatures is None else temperatures.to(f64)
        n_slots = 1 + temps.shape[0]
        i, j, k = torch.meshgrid(*(torch.arange(n, device=dev) for n in (n1, n2, n3)), indexing="ij")
        cell = torch.stack([i.reshape(-1), j.reshape(-1), k.reshape(-1)], 1)  # [n_q, 3], q index order
        size = torch.tensor([n1, n2, n3], device=dev)
        v = ((cell[:, None, None, :] + tetrahedra.long()[None]) % size).reshape(-1, 4, 3)  # [6 N, 4, 3] corners q1
        q1 = (v[..., 0] * n2 + v[..., 1]) * n3 + v[..., 2]
        tets_per_chunk = max(1, self.jdos_chunk_items // max(1, n_band * n_band))
        keep = nu >= cutoff_thz
        occ = occupations(torch.where(keep, nu, 1.0), temps).reshape(n_q * n_band, -1)  # [N band, T]
        band = torch.arange(n_band, device=dev)
        result = torch.zeros(len(targets), n_slots, 3, omega.shape[1], dtype=f64, device=dev)
        for ti, tq in enumerate(targets.long().tolist()):
            tc = torch.tensor([tq // (n2 * n3), (tq // n3) % n2, tq % n3], device=dev)
            v2 = (tc - v) % size
            q2 = (v2[..., 0] * n2 + v2[..., 1]) * n3 + v2[..., 2]
            ws, order = torch.sort(omega[ti].to(f64))
            n_f = ws.shape[0]
            acc = torch.zeros(3, n_f, n_slots, dtype=f64, device=dev)
            for s in range(0, q1.shape[0], tets_per_chunk):
                # items (tetrahedron, l1, l2): flat (q, band) indices of the corners [M, 4]
                ia = (q1[s : s + tets_per_chunk, None, None, :] * n_band + band[None, :, None, None]).expand(
                    -1, n_band, n_band, 4).reshape(-1, 4)
                ib = (q2[s : s + tets_per_chunk, None, None, :] * n_band + band[None, None, :, None]).expand(
                    -1, n_band, n_band, 4).reshape(-1, 4)
                a, b = nu.view(-1)[ia], nu.view(-1)[ib]
                m = keep.view(-1)[ia] & keep.view(-1)[ib]
                live = m.any(1)
                ia, ib, a, b, m = ia[live], ib[live], a[live], b[live], m[live]
                for term, f in ((0, b - a), (1, a - b), (2, a + b)):
                    f, idx = torch.sort(f, dim=1)
                    lo = torch.searchsorted(ws, f[:, 0].contiguous())
                    hi = torch.searchsorted(ws, f[:, 3].contiguous())
                    cnt = hi - lo
                    hit = cnt > 0
                    if not bool(hit.any()):
                        continue
                    f, idx, lo, cnt = f[hit], idx[hit], lo[hit], cnt[hit]
                    na, nb = occ[torch.gather(ia[hit], 1, idx)], occ[torch.gather(ib[hit], 1, idx)]  # [H, 4, T]
                    fac = na - nb if term == 0 else (nb - na if term == 1 else na + nb + 1.0)
                    c = torch.cat([torch.ones_like(f)[..., None], fac], -1) * torch.gather(m[hit], 1, idx)[..., None]
                    item = torch.repeat_interleave(torch.arange(f.shape[0], device=dev), cnt)
                    start = torch.cumsum(cnt, 0) - cnt
                    wi = lo[item] + torch.arange(item.numel(), device=dev) - start[item]
                    wt = tetrahedron_weights(f[item], ws[wi])[2]  # [P, 4]
                    acc[term].index_add_(0, wi, (wt[:, :, None] * c[item]).sum(1))
            inv = torch.empty_like(order)
            inv[order] = torch.arange(n_f, device=dev)
            result[ti] = (acc[:, inv] / (6.0 * n_q)).permute(2, 0, 1)
        return result
