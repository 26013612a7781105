"""fp64 torch specifications of ``chg_phonon_interaction`` and ``chg_imag_self_energy`` with the arguments of
``CudaKernels.phonon_interaction`` and ``CudaKernels.imag_self_energy``.

``ThreePhononSpecKernels`` adds them to ``PhononSpecKernels`` (oracle/phonons.py), so that
``Phonons(..., fc3=..., device="cpu", kernels=ThreePhononSpecKernels())`` runs ``linewidths`` and
``thermal_conductivity`` on the host.  ``interaction_strengths`` evaluates P for explicit (q, q1, q2), q2 not
necessarily reduced, and ``vertex_weights`` the tetrahedron weights of each vertex q1; both are module functions so
that the tests can use them on their own.  ``axes_reversed=True`` plants the bug the non-cubic meshes must catch: every
mesh index is split into coordinates as if the mesh were (n3, n2, n1), which changes nothing on a cubic mesh.
"""
from __future__ import annotations

import math

import torch

from chgnet_b200.phonons import DISPLACEMENT_A2_AMU_THZ, H_EV_PER_THZ
from oracle.joint_dos import occupations
from oracle.phonon_dos import tetrahedron_weights
from oracle.phonons import PhononSpecKernels


def image_averages(img_ptr, img_vec, n_prim, n_super, q):
    """[Q, n_prim, n_super] complex128 rho_kj(q) = (1/m_kj) sum over the minimum images v of pair (k, j) of
    e^{2 pi i q.v}, for reduced ``q`` [Q, 3]."""
    ptr = img_ptr.long()
    counts = ptr[1:] - ptr[:-1]
    pair = torch.repeat_interleave(torch.arange(n_prim * n_super, device=q.device), counts)
    phase = 2 * math.pi * (q.to(torch.float64) @ img_vec.to(torch.float64).T)
    e = torch.complex(torch.cos(phase), torch.sin(phase))
    out = torch.zeros(q.shape[0], n_prim * n_super, dtype=torch.complex128, device=q.device).index_add_(1, pair, e)
    return (out / counts.clamp_min(1).to(torch.float64)).view(q.shape[0], n_prim, n_super)


def interaction_strengths(fc3, img_ptr, img_vec, s2p, inv_sqrt_m, frac, n_mesh, cutoff_thz, q, nu, e, q1, nu1, e1, q2,
                          nu2, e2, phase_sign=1.0):
    """P [Q1, 3n, 3n, 3n] (eV^2) of the target q [3] (frequencies nu [3n], mode-major eigenvectors e [mode, 3n]) with
    the pairs (q1 [Q1, 3], q2 [Q1, 3]) and their modes (nu1, nu2 [Q1, 3n], e1, e2 [Q1, mode, 3n]), G = q - q1 - q2:

        R = e^{-2 pi i G.x_k} sum_{j' in k', j'' in k''} fc3[k, j', j'', a, b, c] rho_kj'(q1) rho_kj''(q2)
        P = C^3 / (36 n_mesh nu nu1 nu2) |sum e*(q) e(q1) e(q2) R / sqrt(m m' m'')|^2

        with C = ``DISPLACEMENT_A2_AMU_THZ`` and P = 0 when a frequency is below ``cutoff_thz``.  ``phase_sign`` -1
        flips the sign of the G phase (the tests show that P then depends on G)."""
    f64, c128 = torch.float64, torch.complex128
    dev = fc3.device
    n_prim, n_super = fc3.shape[0], fc3.shape[1]
    nb = 3 * n_prim
    m = inv_sqrt_m.to(f64)
    g = q.to(f64)[None] - q1.to(f64) - q2.to(f64)
    r1 = image_averages(img_ptr, img_vec, n_prim, n_super, q1)
    r2 = image_averages(img_ptr, img_vec, n_prim, n_super, q2)
    onehot = (s2p.long()[None, :] == torch.arange(n_prim, device=dev)[:, None]).to(f64) * m[s2p.long()][None, :]
    fc = fc3.to(c128).reshape(n_prim, n_super, n_super, 27)
    x = torch.einsum("kjlx,qkl,ml->qkjmx", fc, r2, onehot.to(c128))  # [Q1, k, j', k'', abc]
    r = torch.einsum("qkj,pj,qkjmx->qkpmx", r1, onehot.to(c128), x)  # [Q1, k, k', k'', abc]
    phase = torch.exp(-phase_sign * 2j * math.pi * (g @ frac.to(f64).T)) * m[None, :]  # [Q1, k]
    r = (r * phase[:, :, None, None, None]).reshape(-1, n_prim, n_prim, n_prim, 3, 3, 3)
    r = r.permute(0, 1, 4, 2, 5, 3, 6).reshape(-1, nb, nb, nb)
    t = torch.einsum("la,qabc->qlbc", e.to(c128).conj(), r)
    t = torch.einsum("qmb,qlbc->qlmc", e1.to(c128), t)
    t = torch.einsum("qnc,qlmc->qlmn", e2.to(c128), t)
    nu, nu1, nu2 = nu.to(f64), nu1.to(f64), nu2.to(f64)
    keep = (nu >= cutoff_thz)[None, :, None, None] & (nu1 >= cutoff_thz)[:, None, :, None] & (
        nu2 >= cutoff_thz)[:, None, None, :]
    den = nu[None, :, None, None] * nu1[:, None, :, None] * nu2[:, None, None, :]
    scale = DISPLACEMENT_A2_AMU_THZ**3 / (36.0 * n_mesh)
    return torch.where(keep, scale * (t.real**2 + t.imag**2) / torch.where(keep, den, 1.0), 0.0)


def _mesh_coords(i, mesh, axes_reversed=False):
    """The coordinates [..., 3] of the mesh indices ``i``; ``axes_reversed`` splits with (n3, n2, n1) instead and wraps
    the result onto the mesh (the planted bug)."""
    n1, n2, n3 = mesh[::-1] if axes_reversed else mesh
    c = torch.stack([i // (n2 * n3), (i // n3) % n2, i % n3], -1)
    return c % torch.tensor(mesh, device=c.device) if axes_reversed else c


def _mesh_index(c, mesh):
    return (c[..., 0] * mesh[1] + c[..., 1]) * mesh[2] + c[..., 2]


def vertex_weights(freqs, mesh, tetrahedra, target, omega, q1, cutoff_thz, chunk_items=1 << 14, axes_reversed=False):
    """[Q1, l, l1, l2, 3]: the weights (g2, g1+, g1-) with which vertex q1 (mesh indices ``q1`` [Q1]) enters the
    tetrahedron averages of d(w - nu1 - nu2), d(w + nu1 - nu2) and d(w - nu1 + nu2) at w = omega[l]: 1/6 of the sum
    over the 24 (tetrahedron, corner) whose corner is q1 of ``tetrahedron_weights``' weight of that corner, the corner
    values nu1 + nu2, nu2 - nu1 and nu1 - nu2 at every corner q1' (nu1 = freqs[q1', l1], nu2 = freqs[target - q1',
    l2]).  0 where nu1(q1) or nu2(q - q1) is below ``cutoff_thz``, or omega[l] is."""
    f64 = torch.float64
    dev = freqs.device
    mesh = tuple(int(n) for n in mesh)
    size = torch.tensor(mesh, device=dev)
    nu = freqs.to(f64)
    n_q1, nb = q1.shape[0], nu.shape[1]
    om = omega.to(f64)
    tgt = _mesh_coords(torch.tensor(int(target), device=dev), mesh, axes_reversed)
    c1 = _mesh_coords(q1.long(), mesh, axes_reversed)  # [Q1, 3]
    off = tetrahedra.long()  # [6, 4, 3]
    # corners of the 24 (tetrahedron t, corner v) around each q1: cell = q1 - off[t, v], corners cell + off[t, u]
    corners = (c1[:, None, None, None, :] - off[:, :, None, :][None] + off[:, None, :, :][None]) % size  # [Q1,6,4,4,3]
    qa = _mesh_index(corners, mesh).reshape(n_q1, 24, 4)
    qb = _mesh_index((tgt - corners) % size, mesh).reshape(n_q1, 24, 4)
    own = torch.arange(24, device=dev) % 4  # the corner v that is q1
    out = torch.zeros(n_q1 * nb * nb, nb, 3, dtype=f64, device=dev)
    items = torch.arange(n_q1 * nb * nb, device=dev)
    for s in range(0, items.numel(), chunk_items):
        it = items[s : s + chunk_items]
        qi, l1, l2 = it // (nb * nb), (it // nb) % nb, it % nb
        a = nu[qa[qi], l1[:, None, None]]  # [M, 24, 4]
        b = nu[qb[qi], l2[:, None, None]]
        live = (a[:, 0, own[0]] >= cutoff_thz) & (b[:, 0, own[0]] >= cutoff_thz)  # nu1, nu2 at q1 itself
        for cls, f in enumerate((a + b, b - a, a - b)):
            fs, idx = torch.sort(f, dim=-1)
            pos = torch.argmax((idx == own[None, :, None]).to(torch.int8), dim=-1)  # [M, 24]
            hit = (om[None, None, :] >= fs[..., :1]) & (om[None, None, :] < fs[..., 3:]) & (om >= cutoff_thz)
            hit &= live[:, None, None]
            mi, ti, li = torch.nonzero(hit, as_tuple=True)
            if mi.numel() == 0:
                continue
            wt = tetrahedron_weights(fs[mi, ti], om[li])[2]  # [H, 4]
            w = torch.gather(wt, 1, pos[mi, ti][:, None])[:, 0] / 6.0
            flat = torch.zeros(it.numel() * nb, dtype=f64, device=dev).index_add_(0, mi * nb + li, w)
            out[s : s + it.numel(), :, cls] = flat.view(-1, nb)
    return out.view(n_q1, nb, nb, nb, 3).permute(0, 3, 1, 2, 4)


class ThreePhononSpecKernels(PhononSpecKernels):
    """``PhononSpecKernels`` with the specifications of the two three-phonon kernels; ``axes_reversed=True`` plants
    the axis-reversed split of ``_mesh_coords`` in every kernel of this class and its subclasses."""

    # fc3-by-q1 work per chunk of the interaction specification (complex128 elements of its largest intermediate)
    ph3_chunk_elems = 1 << 22
    # (q1, l1, l2) items per chunk of the vertex weights
    ise_chunk_items = 1 << 14

    def __init__(self, *, axes_reversed: bool = False):
        self.axes_reversed = axes_reversed

    def phonon_interaction(self, fc3, img_ptr, img_vec, s2p, inv_sqrt_m, frac, mesh, freqs, eigvecs, target, q1,
                           cutoff_thz, out):
        """out [Q1, 3n, 3n, 3n] = ``interaction_strengths`` of the mesh index ``target`` with the mesh indices
        ``q1`` and q2 = target - q1 on the mesh (reduced coordinates i / n)."""
        dev = freqs.device
        mesh = tuple(int(n) for n in mesh)
        size = torch.tensor(mesh, device=dev)
        n_mesh = mesh[0] * mesh[1] * mesh[2]
        n_prim, n_super = fc3.shape[0], fc3.shape[1]
        tc = _mesh_coords(torch.tensor(int(target), device=dev), mesh, self.axes_reversed)
        c1 = _mesh_coords(q1.long(), mesh, self.axes_reversed)
        c2 = (tc - c1) % size
        i2 = _mesh_index(c2, mesh)
        chunk = max(1, self.ph3_chunk_elems // (n_prim * n_super * n_prim * 27))
        for s in range(0, q1.shape[0], chunk):
            sl = slice(s, s + chunk)
            a, b = q1.long()[sl], i2[sl]
            out[sl] = interaction_strengths(fc3, img_ptr, img_vec, s2p, inv_sqrt_m, frac, n_mesh, cutoff_thz,
                                            tc.to(torch.float64) / size, freqs[int(target)], eigvecs[int(target)],
                                            c1[sl].to(torch.float64) / size, freqs[a], eigvecs[a],
                                            c2[sl].to(torch.float64) / size, freqs[b], eigvecs[b])

    def imag_self_energy(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, gamma):
        """gamma[t, l] += 18 pi / h^2 sum_{q1, l1, l2} p[q1, l, l1, l2] [(1 + n1 + n2) g2 + (n1 - n2) (g1+ - g1-)] with
        the ``vertex_weights`` (g2, g1+, g1-), n1 = n(freqs[q1, l1]), n2 = n(freqs[target - q1, l2]) the
        ``occupations`` at temperatures[t]."""
        f64 = torch.float64
        dev = freqs.device
        mesh_t = tuple(int(n) for n in mesh)
        size = torch.tensor(mesh_t, device=dev)
        nu = freqs.to(f64)
        w = vertex_weights(nu, mesh_t, tetrahedra, target, omega, q1, cutoff_thz, self.ise_chunk_items,
                           self.axes_reversed)
        tc = _mesh_coords(torch.tensor(int(target), device=dev), mesh_t, self.axes_reversed)
        i2 = _mesh_index((tc - _mesh_coords(q1.long(), mesh_t, self.axes_reversed)) % size, mesh_t)
        nu1, nu2 = nu[q1.long()], nu[i2]  # [Q1, nb]
        n1 = occupations(torch.where(nu1 >= cutoff_thz, nu1, 1.0), temperatures)  # [Q1, nb, T]
        n2 = occupations(torch.where(nu2 >= cutoff_thz, nu2, 1.0), temperatures)
        s2 = n1[:, :, None, :] + n2[:, None, :, :]  # [Q1, l1, l2, T]
        d1 = n1[:, :, None, :] - n2[:, None, :, :]
        g2 = torch.einsum("qlab,qabt->tl", p.to(f64) * w[..., 0], 1.0 + s2)
        g1 = torch.einsum("qlab,qabt->tl", p.to(f64) * (w[..., 1] - w[..., 2]), d1)
        gamma += (18.0 * math.pi / H_EV_PER_THZ**2) * (g2 + g1)
