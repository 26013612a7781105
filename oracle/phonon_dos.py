"""TEST INFRASTRUCTURE — phonon group velocities and densities of states: the specifications of
``chg_dynamical_matrix_derivatives`` and ``chg_tetrahedron_dos``.

* ``PhononDosSpecKernels``: ``PhononSpecKernels`` (oracle/phonons.py) plus fp64 torch specifications of the two kernels
  with the arguments of ``CudaKernels``, so that ``Phonons(..., device="cpu", kernels=PhononDosSpecKernels())`` runs
  ``group_velocities`` and ``dos`` on the host.
* ``tetrahedron_weights``: the linear tetrahedron closed forms for one (tetrahedron, band), vectorised.

Never imported by the product path.
"""
from __future__ import annotations

import math

import torch

from oracle.phonons import PhononSpecKernels


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


class PhononDosSpecKernels(PhononSpecKernels):
    """fp64 specifications of the phonon kernels, group-velocity and DOS kernels included."""

    # (tetrahedron, band) pairs per chunk of the DOS specification
    dos_chunk_pairs = 1 << 16

    def dynamical_matrix_derivatives(self, fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, prim_lattice, ddyn):
        """ddyn[q, c] = the Hermitian part of dD/dQ_c: the sum of ``dynamical_matrices`` with each image term
        multiplied by 2 pi i r_c, r = img_vec @ prim_lattice."""
        f64 = torch.float64
        n_prim, n_super = fc.shape[0], fc.shape[1]
        ptr = img_ptr.long()
        counts = ptr[1:] - ptr[:-1]
        pair_of_image = torch.repeat_interleave(torch.arange(n_prim * n_super, device=fc.device), counts)
        w = (1.0 / counts.to(f64))[pair_of_image]
        r = img_vec.to(f64) @ prim_lattice.to(f64)  # [n_img, 3] Cartesian, A
        m = inv_sqrt_m.to(f64)
        scale = (m[:, None] * m[None, :]).repeat_interleave(3, 0).repeat_interleave(3, 1)
        chunk = max(1, self.chunk_elems // max(1, n_prim * n_super))
        for s in range(0, qpoints.shape[0], chunk):
            q = qpoints[s : s + chunk].to(f64)
            phase = 2 * math.pi * (q @ img_vec.to(f64).T)  # [Qc, n_img]
            e = torch.complex(torch.cos(phase), torch.sin(phase)) * w
            for c in range(3):
                ec = e * (2j * math.pi * r[:, c])
                pair = torch.zeros(q.shape[0], n_prim * n_super, dtype=torch.complex128, device=fc.device)
                pair.index_add_(1, pair_of_image, ec)
                blocks = pair.view(-1, n_prim, n_super, 1, 1) * fc.to(torch.complex128)[None]
                d = torch.zeros(q.shape[0], n_prim, n_prim, 3, 3, dtype=torch.complex128, device=fc.device)
                d.index_add_(2, s2p.long(), blocks)
                d = d.permute(0, 1, 3, 2, 4).reshape(q.shape[0], 3 * n_prim, 3 * n_prim) * scale
                ddyn[s : s + chunk, c] = 0.5 * (d + d.conj().transpose(1, 2))

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
