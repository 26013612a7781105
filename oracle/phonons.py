"""TEST INFRASTRUCTURE — phonons: the fp64 specifications of the phonon kernels and the oracle force constants.

* ``PhononSpecKernels``: fp64 torch specifications of ``chg_dynamical_matrices``, ``chg_dynamical_matrix_derivatives``,
  ``chg_tetrahedron_dos``, ``chg_thermal_displacements`` and ``chg_joint_dos`` with the arguments of ``CudaKernels``,
  so that ``Phonons(..., device="cpu", kernels=PhononSpecKernels())`` runs every ``Phonons`` method on the host.  D(q)
  and dD/dQ are explicit sums over (primitive atom, supercell atom) pairs and their minimum images, chunked over q.
  Unlike the kernel, the joint-DOS specification evaluates both class-1 terms, d(w + nu1 - nu2) and d(w - nu1 + nu2),
  separately.
* ``oracle_compact_fcs``: the compact force constants of ``oracle/chgnet_oracle.py`` on a supercell, from
  ``oracle_hvp`` with the 3 n_prim unit directions on the ``p2s`` atoms.

The closed forms the specifications evaluate are module functions of their own: ``tetrahedron_weights``
(oracle/phonon_dos.py), ``mode_weights`` (oracle/thermal_displacements.py) and ``occupations`` (oracle/joint_dos.py).

Never imported by the product path.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.hessian import oracle_hvp
from oracle.joint_dos import occupations
from oracle.phonon_dos import tetrahedron_weights
from oracle.thermal_displacements import VOIGT, mode_weights


def _images(fc, img_ptr, inv_sqrt_m):
    """The pair (k N + j) of every minimum image, its weight 1 / multiplicity, and the [3n, 3n] mass scale
    inv_sqrt_m[k] inv_sqrt_m[k'] of D."""
    n_prim, n_super = fc.shape[0], fc.shape[1]
    ptr = img_ptr.long()
    counts = ptr[1:] - ptr[:-1]
    pair_of_image = torch.repeat_interleave(torch.arange(n_prim * n_super, device=fc.device), counts)
    w = (1.0 / counts.to(torch.float64))[pair_of_image]
    m = inv_sqrt_m.to(torch.float64)
    scale = (m[:, None] * m[None, :]).repeat_interleave(3, 0).repeat_interleave(3, 1)
    return pair_of_image, w, scale


def _hermitian_part(e, pair_of_image, fc, s2p, scale):
    """(D + D^H)/2 [Qc, 3n, 3n] of the image terms e [Qc, n_img]: summed over the images of each pair, times fc,
    summed over the supercell atoms j of each k', times the mass scale."""
    n_prim, n_super = fc.shape[0], fc.shape[1]
    pair = torch.zeros(e.shape[0], n_prim * n_super, dtype=torch.complex128, device=fc.device)
    pair.index_add_(1, pair_of_image, e)
    blocks = pair.view(-1, n_prim, n_super, 1, 1) * fc.to(torch.complex128)[None]  # [Qc, k, j, a, b]
    d = torch.zeros(e.shape[0], n_prim, n_prim, 3, 3, dtype=torch.complex128, device=fc.device)
    d.index_add_(2, s2p.long(), blocks)
    d = d.permute(0, 1, 3, 2, 4).reshape(e.shape[0], 3 * n_prim, 3 * n_prim) * scale
    return 0.5 * (d + d.conj().transpose(1, 2))


class PhononSpecKernels:
    """fp64 specifications of the phonon kernels."""

    # pair-by-q work per chunk (complex128 elements of the [q, pair] phase sums)
    chunk_elems = 1 << 22
    # (tetrahedron, band) pairs per chunk of the DOS specification
    dos_chunk_pairs = 1 << 16
    # (q, mode) pairs per chunk of the thermal-displacement specification
    td_chunk_pairs = 1 << 14
    # (tetrahedron, band pair) items per chunk of the joint-DOS specification
    jdos_chunk_items = 1 << 17

    def dynamical_matrices(self, fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, dyn):
        """dyn[q, 3k+a, 3k'+b] = (D + D^H)/2 with D = sum_{j: s2p[j]=k'} fc[k,j,a,b] (1/m_kj) sum_v e^{2 pi i q.v}
        inv_sqrt_m[k] inv_sqrt_m[k']."""
        f64 = torch.float64
        pair_of_image, w, scale = _images(fc, img_ptr, inv_sqrt_m)
        chunk = max(1, self.chunk_elems // max(1, fc.shape[0] * fc.shape[1]))
        for s in range(0, qpoints.shape[0], chunk):
            q = qpoints[s : s + chunk].to(f64)
            phase = 2 * math.pi * (q @ img_vec.to(f64).T)  # [Qc, n_img]
            e = torch.complex(torch.cos(phase), torch.sin(phase)) * w
            dyn[s : s + chunk] = _hermitian_part(e, pair_of_image, fc, s2p, scale)

    def dynamical_matrix_derivatives(self, fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, prim_lattice, ddyn):
        """ddyn[q, c] = the Hermitian part of dD/dQ_c: the sum of ``dynamical_matrices`` with each image term
        multiplied by 2 pi i r_c, r = img_vec @ prim_lattice."""
        f64 = torch.float64
        pair_of_image, w, scale = _images(fc, img_ptr, inv_sqrt_m)
        r = img_vec.to(f64) @ prim_lattice.to(f64)  # [n_img, 3] Cartesian, A
        chunk = max(1, self.chunk_elems // max(1, fc.shape[0] * fc.shape[1]))
        for s in range(0, qpoints.shape[0], chunk):
            q = qpoints[s : s + chunk].to(f64)
            phase = 2 * math.pi * (q @ img_vec.to(f64).T)  # [Qc, n_img]
            e = torch.complex(torch.cos(phase), torch.sin(phase)) * w
            for c in range(3):
                ddyn[s : s + chunk, c] = _hermitian_part(e * (2j * math.pi * r[:, c]), pair_of_image, fc, s2p, scale)

    def tetrahedron_dos(self, freqs, mesh, tetrahedra, omega, dos, idos, proj=None, pdos=None):
        """dos[f] = sum g_T(omega_f), idos[f] = sum n_T(omega_f), pdos[s, f] = sum_T sum_i wt_T,i(omega_f)
        proj[q_i, band, s], over every (tetrahedron T, band) of the mesh, each weighted 1 / (6 n_q).  Only the
        frequency points inside [e0, e3) of a pair are evaluated; those at or above e3 add n = 1."""
        f64 = torch.float64
        n1, n2, n3 = (int(n) for n in mesh)
        n_q, n_band = freqs.shape
        dev = freqs.device
        ws, order = torch.sort(omega.to(f64))
        n_f = ws.shape[0]
        acc_g = torch.zeros(n_f, dtype=f64, device=dev)
        acc_n = torch.zeros(n_f + 1, dtype=f64, device=dev)  # +1 from the first point >= e3 on (a cumulative sum)
        acc_in = torch.zeros(n_f, dtype=f64, device=dev)
        acc_p = torch.zeros(n_f, proj.shape[2] if proj is not None else 0, dtype=f64, device=dev)
        i, j, k = torch.meshgrid(*(torch.arange(n, device=dev) for n in (n1, n2, n3)), indexing="ij")
        cell = torch.stack([i.reshape(-1), j.reshape(-1), k.reshape(-1)], 1)  # [n_q, 3], q index order
        off = tetrahedra.long()  # [6, 4, 3]
        size = torch.tensor([n1, n2, n3], device=dev)
        cells_per_chunk = max(1, self.dos_chunk_pairs // (6 * max(n_band, 1)))
        for s in range(0, n_q, cells_per_chunk):
            v = (cell[s : s + cells_per_chunk, None, None, :] + off[None]) % size  # [C, 6, 4, 3]
            qv = ((v[..., 0] * n2 + v[..., 1]) * n3 + v[..., 2]).reshape(-1, 4)  # [T, 4]
            e = freqs.to(f64)[qv].permute(0, 2, 1).reshape(-1, 4)  # [T n_band, 4], band fastest
            qv = qv[:, None, :].expand(-1, n_band, 4).reshape(-1, 4)
            band = torch.arange(n_band, device=dev).repeat(qv.shape[0] // n_band)
            e, idx = torch.sort(e, dim=1)
            qv = torch.gather(qv, 1, idx)
            lo = torch.searchsorted(ws, e[:, 0].contiguous())
            hi = torch.searchsorted(ws, e[:, 3].contiguous())
            acc_n += torch.bincount(hi, minlength=n_f + 1).to(f64)
            cnt = hi - lo
            pair = torch.repeat_interleave(torch.arange(e.shape[0], device=dev), cnt)
            if pair.numel() == 0:
                continue
            start = torch.cumsum(cnt, 0) - cnt
            wi = lo[pair] + torch.arange(pair.numel(), device=dev) - start[pair]
            n, g, wt = tetrahedron_weights(e[pair], ws[wi])
            acc_g.index_add_(0, wi, g)
            acc_in.index_add_(0, wi, n)
            if proj is not None:
                p = proj.to(f64)[qv[pair], band[pair, None]]  # [M, 4, S]
                acc_p.index_add_(0, wi, (wt[:, :, None] * p).sum(1))
        scale = 1.0 / (6.0 * n_q)
        inv = torch.empty_like(order)
        inv[order] = torch.arange(n_f, device=dev)
        dos.copy_((acc_g * scale)[inv])
        idos.copy_(((torch.cumsum(acc_n, 0)[:n_f] + acc_in) * scale)[inv])
        if proj is not None:
            pdos.copy_((acc_p * scale)[inv].T)

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


def oracle_compact_fcs(weights: dict, graph, p2s, args=None) -> np.ndarray:
    """[n_prim, N, 3, 3] Phi[k, j, a, b] = (H e_{p2s[k], a})[j, b] of the oracle in fp64, H the Hessian of ``graph``
    (the supercell)."""
    n = graph.atomic_number.shape[0]
    n_prim = len(p2s)
    v = torch.zeros(n_prim, 3, n, 3, dtype=torch.float64)
    for a in range(3):
        v[torch.arange(n_prim), a, torch.as_tensor(np.asarray(p2s)).long(), a] = 1.0
    hv = oracle_hvp(weights, [graph] * (3 * n_prim), v.reshape(3 * n_prim * n, 3), args)
    return hv.reshape(n_prim, 3, n, 3).permute(0, 2, 1, 3).contiguous().numpy()
