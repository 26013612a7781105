"""Crystals and analytic potentials for the effective force constant tests: fcc nearest-neighbour springs with an
optional quartic bond term, and harmonic surrogates F = F_0 - Phi_sc u of given force constants."""
import numpy as np
import torch

from chgnet_b200.phonons import _expand_compact, acoustic_sum_rule, make_supercell, translation_table

# fcc aluminium-like: primitive vectors (0, h, h), (h, 0, h), (h, h, 0), one atom of Z = 13
FCC_H, FCC_Z = 2.0, 13
FCC_LATTICE = FCC_H * (np.ones((3, 3)) - np.eye(3))
# the conventional cube in primitive vectors, and twice it (32 atoms, a non-diagonal M)
FCC_CONV = np.array([[-1, 1, 1], [1, -1, 1], [1, 1, -1]])
# the six nearest-neighbour vectors of one sign, in primitive fractional coordinates
FCC_NN = np.array([[1, 0, 0], [0, 1, 0], [0, 0, 1], [1, -1, 0], [0, 1, -1], [1, 0, -1]])


def fcc_bonds(sc):
    """(i [B], j [B], e_hat [B, 3]): every nearest-neighbour bond of the fcc supercell once (6 per atom)."""
    inv_m = np.linalg.inv(sc.matrix.astype(np.float64))
    i_all, j_all, e_all = [], [], []
    for i in range(len(sc.z)):
        for n in FCC_NN:
            x = (sc.frac[i] + n @ inv_m) % 1.0
            j = int(np.argmin(np.abs((sc.frac - x + 0.5) % 1.0 - 0.5).sum(1)))
            r = n @ FCC_LATTICE
            i_all.append(i), j_all.append(j), e_all.append(r / np.linalg.norm(r))
    return np.array(i_all), np.array(j_all), np.array(e_all)


def fcc_springs(m, k):
    """The fcc supercell ``m`` and the compact force constants of central nearest-neighbour springs k (eV/A^2)."""
    sc = make_supercell([FCC_Z], np.zeros((1, 3)), FCC_LATTICE, m)
    i, j, e = fcc_bonds(sc)
    full = np.zeros((len(sc.z), len(sc.z), 3, 3))
    for a, b, eh in zip(i, j, e):
        p = k * np.outer(eh, eh)
        full[a, b] -= p
        full[b, a] -= p
        full[a, a] += p
        full[b, b] += p
    return sc, np.ascontiguousarray(full[sc.p2s])


class QuarticSprings:
    """forces(frac) of fcc nearest-neighbour bonds with energy k/2 s^2 + lam/4 s^4 each, s = e_hat . (u_j - u_i) the
    linearised stretch, u the displacement from the supercell's positions.  ``keep`` stores every call's (frac, F)."""

    def __init__(self, sc, k, lam, keep=False):
        self.sc, self.k, self.lam = sc, k, lam
        self.i, self.j, self.e = fcc_bonds(sc)
        self.ref = np.asarray(sc.frac, dtype=np.float32).astype(np.float64)
        self.calls = [] if keep else None

    def __call__(self, frac):
        x = frac.cpu().numpy()
        u = (x - self.ref[None]) @ self.sc.lattice
        s = np.einsum("mbx,bx->mb", u[:, self.j] - u[:, self.i], self.e)
        de = self.k * s + self.lam * s**3
        f = np.zeros_like(u)
        for m in range(len(u)):
            np.add.at(f[m], self.i, de[m][:, None] * self.e)
            np.add.at(f[m], self.j, -de[m][:, None] * self.e)
        en = (0.5 * self.k * s**2 + 0.25 * self.lam * s**4).sum(1)
        if self.calls is not None:
            self.calls.append((x, f))
        return torch.from_numpy(f), torch.from_numpy(en)


class HarmonicSurrogate:
    """forces(frac) = F_0 - Phi_sc u of the compact force constants ``fc`` (after the acoustic sum rule), with the
    residual forces ``f0`` [N, 3] and energy E_0 + (-F_0 . u + u Phi_sc u / 2)."""

    def __init__(self, sc, fc, f0, e0=-3.0):
        perm = translation_table(sc)
        inv = np.empty_like(perm)
        np.put_along_axis(inv, perm, np.arange(len(sc.z))[None].repeat(len(perm), 0), axis=1)
        phi = torch.as_tensor(acoustic_sum_rule(np.asarray(fc, dtype=np.float64), sc.p2s)[0])
        self.phi_sc = _expand_compact(phi, torch.as_tensor(inv.astype(np.int64))).numpy()
        self.sc, self.f0, self.e0 = sc, np.asarray(f0, dtype=np.float64), e0
        self.ref = np.asarray(sc.frac, dtype=np.float32).astype(np.float64)

    def __call__(self, frac):
        x = frac.cpu().numpy()
        u = ((x - self.ref[None]) @ self.sc.lattice).reshape(len(x), -1)
        f = self.f0.reshape(1, -1) - u @ self.phi_sc.T
        en = self.e0 - u @ self.f0.reshape(-1) + 0.5 * np.einsum("mi,ij,mj->m", u, self.phi_sc, u)
        return torch.from_numpy(f.reshape(x.shape)), torch.from_numpy(en)
