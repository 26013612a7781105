"""Harmonic phonons from supercell force constants (``CHGNet.phonons``).

* ``make_supercell``: the supercell of a primitive cell for an integer matrix M (lattice ``M @ lattice``, rows are
  lattice vectors, as phonopy builds it), its atom maps and the minimum-image table of every (primitive atom,
  supercell atom) pair.
* ``compact_force_constants``: the force constants ``[n_prim, N_super, 3, 3]`` (phonopy's compact layout) from the
  3 n_prim Hessian-vector products that move the atoms of one primitive cell.  The supercell is periodic in the
  primitive lattice, Phi(k l, k' l') = Phi(k 0, k' (l' - l)), so these columns determine every force constant.
* ``Phonons``: dynamical matrices D(q) on the device (``chg_dynamical_matrices``, csrc/phonons.cu), frequencies and
  eigenvectors by ``torch.linalg.eigh``, and harmonic thermodynamics on a Gamma-centred mesh; group velocities from
  dD/dQ (``chg_dynamical_matrix_derivatives``) and the linear tetrahedron density of states, total and projected on
  atoms (``chg_tetrahedron_dos``); anisotropic thermal displacement matrices U(T) on a mesh
  (``chg_thermal_displacements``), Cartesian and in the CIF convention (``cif_displacement_matrices``); two-phonon
  joint densities of states and their occupation-weighted forms at mesh q-points, and per mode as the three-phonon
  phase space (``chg_joint_dos``); coherent one-phonon neutron structure factors S(Q, omega) per mode at scattering
  vectors and their broadened spectra, per Q (``dynamic_structure_factor``) and averaged over directions for powders
  (``powder_spectrum``), with ``chg_structure_factors`` and ``chg_broadened_spectrum``; with third-order force
  constants (``third_order_force_constants``), three-phonon interaction strengths (``chg_phonon_interaction``),
  linewidths (``chg_imag_self_energy``) and the lattice thermal conductivity in the relaxation-time approximation;
  frequency-resolved self-energies (``chg_self_energy_spectrum``) and anharmonic phonon spectral functions; the Wigner
  coherence term of the thermal conductivity (``chg_coherence_conductivity``); isotope scattering rates
  (``chg_isotope_scattering``, no fc3 needed) and isotope and boundary scattering in every thermal conductivity;
  temperature-dependent effective force constants fitted to the forces of thermally displaced supercells
  (``effective_force_constants``, with ``chg_sample_displacements`` and ``chg_displacement_moments``).

Units: eV/A^2 for force constants, amu for masses, THz for frequencies (imaginary modes as negative numbers),
eV and eV/K per primitive cell for the thermodynamic functions, THz*A (100 m/s) for group velocities, states/THz per
primitive cell for densities of states, A^2 for thermal displacement matrices, 1/THz for joint densities of states,
b^2 per primitive cell for structure factors (b the caller's scattering lengths) and b^2/THz for their spectra,
eV/A^3 for third-order force constants, eV^2 for interaction strengths, THz for linewidths, ps for lifetimes and
W/(m K) for thermal conductivities, 1/THz for spectral functions.
"""
from __future__ import annotations

import itertools
import math
from dataclasses import dataclass

import numpy as np
import torch

from chgnet_b200._lib import (JDOS_MAX_CHUNKS, coherence_scratch_doubles, ise_scratch_doubles, isotope_scratch_doubles,
                              ph3_scratch_doubles, se_scratch_doubles, sqw_scratch_doubles)
from chgnet_b200.dynamics import ATOMIC_MASSES, KB

# sqrt(eV / (A^2 amu)) / 2 pi in THz, CODATA 2018 (phonopy's older constant is 15.633302)
_EV, _AMU, _ANGSTROM, _H = 1.602176634e-19, 1.66053906660e-27, 1e-10, 6.62607015e-34
THZ_PER_SQRT_EV_A2_AMU = math.sqrt(_EV / (_ANGSTROM**2 * _AMU)) / (2 * math.pi) / 1e12
H_EV_PER_THZ = _H / _EV * 1e12  # h nu in eV for nu in THz
# h / k_B in K/THz (the constant of chg_thermal_displacements)
H_OVER_KB_K_PER_THZ = H_EV_PER_THZ / KB
# hbar / (2 m omega) = C / (m [amu] nu [THz]) in A^2: C = h / (8 pi^2 amu 1 THz) = 0.5053790 A^2
DISPLACEMENT_A2_AMU_THZ = _H / (8 * math.pi**2 * _AMU * 1e12) / _ANGSTROM**2
# image lengths within this of the shortest count as minimum images (A)
IMAGE_TOL = 1e-5
# modes below this |nu| (THz) are left out of the thermodynamic sums
THERMAL_CUTOFF_THZ = 1e-3
# adjacent modes closer than this (THz) form a degenerate set for the group velocities
DEGENERACY_THZ = 1e-4
# eV THz / (K A) in W/(m K): the unit of C v v tau / V with C in eV/K, v in THz A, tau in ps and V in A^3
KAPPA_W_PER_MK = _EV * 1e12 / _ANGSTROM


def supercell_matrix(m) -> np.ndarray:
    """[3,3] integer matrix from a 3x3 matrix or a 3-vector (diagonal); raises ValueError if it is not integral or
    its determinant is not positive."""
    a = np.asarray(m, dtype=np.float64)
    if a.shape == (3,):
        a = np.diag(a)
    if a.shape != (3, 3):
        raise ValueError(f"supercell_matrix must be a 3x3 matrix or a 3-vector, got shape {list(a.shape)}")
    if not np.all(np.isfinite(a)) or np.any(a != np.round(a)):
        raise ValueError(f"supercell_matrix must be integral, got {a.tolist()}")
    mi = np.round(a).astype(np.int64)
    if round(np.linalg.det(mi)) <= 0:
        raise ValueError(f"supercell_matrix must have a positive determinant, got {mi.tolist()}")
    return mi


def lattice_points(m: np.ndarray) -> np.ndarray:
    """[det M, 3] integer vectors n (primitive fractional coordinates) with n M^-1 in [0,1)^3, origin first."""
    det = int(round(np.linalg.det(m)))
    adj = np.round(np.linalg.inv(m) * det).astype(np.int64)  # det M^-1, integral
    corners = np.array(list(itertools.product((0, 1), repeat=3))) @ m
    axes = [np.arange(corners[:, i].min(), corners[:, i].max() + 1) for i in range(3)]
    n = np.array(np.meshgrid(*axes, indexing="ij")).reshape(3, -1).T
    x = n @ adj  # det * (n M^-1), exact
    n = n[np.all((x >= 0) & (x < det), axis=1)]
    n = n[np.lexsort((n[:, 2], n[:, 1], n[:, 0], np.abs(n).sum(axis=1)))]
    assert len(n) == det and not n[0].any()
    return n


def _reduce_basis(b: np.ndarray) -> np.ndarray:
    """Unimodular U with U b pairwise reduced (|b_i . b_j| <= |b_j|^2 / 2): every step shortens a vector."""
    b, u = b.copy(), np.eye(3, dtype=np.int64)
    for _ in range(1000):
        changed = False
        for i, j in itertools.permutations(range(3), 2):
            mu = int(np.round(b[i] @ b[j] / (b[j] @ b[j])))
            if mu:
                b[i] -= mu * b[j]
                u[i] -= mu * u[j]
                changed = True
        if not changed:
            return u
    raise RuntimeError("supercell basis reduction did not converge")


def minimum_images(frac_sc: np.ndarray, p2s: np.ndarray, m: np.ndarray, lattice: np.ndarray):
    """Minimum images of r_j - r_p2s[k] over the supercell lattice, for every primitive atom k and supercell atom j.

    Returns the CSR ``(img_ptr [n_prim N + 1] int32, img_vec [n_img, 3] fp64)``: the images of pair (k, j) are the rows
    ``img_ptr[k N + j] : img_ptr[k N + j + 1]`` of ``img_vec``, in primitive fractional coordinates, every image whose
    length is within ``IMAGE_TOL`` of the shortest.  The search runs in a reduced supercell basis over every lattice
    vector that could be that short, so skewed supercells lose no image."""
    s = m @ lattice
    u = _reduce_basis(s.astype(np.float64))
    red = u @ s  # reduced supercell basis (Cartesian rows)
    red_m = u @ m  # the same in primitive fractional coordinates
    to_red = np.linalg.inv(u.astype(np.float64))  # supercell frac -> reduced frac
    n_super = len(frac_sc)
    ptr, vecs = [0], []
    d_red = [None] * len(p2s)
    for k, k0 in enumerate(p2s):
        d = (frac_sc - frac_sc[k0]) @ to_red
        d_red[k] = d - np.round(d)  # nearest copy in the reduced cell
    # |m_i| <= (|d'| + |d|) |column i of red^-1| for any image d' = d + m red no longer than d
    longest = max(float(np.linalg.norm(d @ red, axis=1).max()) for d in d_red)
    reach = np.ceil((2 * longest + IMAGE_TOL) * np.linalg.norm(np.linalg.inv(red), axis=0)).astype(int)
    cand = np.array(list(itertools.product(*[range(-r, r + 1) for r in reach])), dtype=np.float64)
    for k in range(len(p2s)):
        v = d_red[k][:, None, :] + cand[None, :, :]  # [N, C, 3] reduced frac
        length = np.linalg.norm(v @ red, axis=2)
        keep = length <= length.min(axis=1, keepdims=True) + IMAGE_TOL
        counts = keep.sum(axis=1)
        vecs.append(v[keep] @ red_m)  # row-major: j ascending, candidates in a fixed order
        ptr.extend(ptr[-1] + np.cumsum(counts))
    img_ptr = np.asarray(ptr, dtype=np.int64)
    assert len(img_ptr) == len(p2s) * n_super + 1
    if img_ptr[-1] >= 2**31:
        raise ValueError("minimum-image table too large")
    return img_ptr.astype(np.int32), np.ascontiguousarray(np.concatenate(vecs), dtype=np.float64)


@dataclass
class Supercell:
    """A supercell in atom-major order: atom j = k n_cells + l sits at r_k + R_l (modulo the supercell lattice)."""

    z: np.ndarray  # [N] int32
    frac: np.ndarray  # [N,3] supercell fractional coordinates, wrapped into [0,1)
    lattice: np.ndarray  # [3,3] M @ primitive lattice
    matrix: np.ndarray  # [3,3] int M
    points: np.ndarray  # [n_cells,3] int lattice points R_l in primitive fractional coordinates, origin first
    s2p: np.ndarray  # [N] primitive atom of each supercell atom
    p2s: np.ndarray  # [n_prim] the l = 0 supercell atom of each primitive atom
    prim_z: np.ndarray
    prim_frac: np.ndarray
    prim_lattice: np.ndarray
    img_ptr: np.ndarray  # minimum-image CSR (minimum_images)
    img_vec: np.ndarray

    @property
    def multiplicities(self) -> np.ndarray:
        """[n_prim, N] number of minimum images of each pair."""
        return np.diff(self.img_ptr).reshape(len(self.p2s), len(self.s2p))


def make_supercell(z, frac, lattice, matrix) -> Supercell:
    """Supercell of the primitive cell ``(z, frac, lattice)`` for the integer ``matrix`` (3x3, or a 3-vector meaning a
    diagonal): lattice ``M @ lattice``; atom j = k n_cells + l is primitive atom k moved by lattice point l."""
    m = supercell_matrix(matrix)
    z = np.asarray(z, dtype=np.int32).reshape(-1)
    frac = np.asarray(frac, dtype=np.float64).reshape(-1, 3)
    lattice = np.asarray(lattice, dtype=np.float64).reshape(3, 3)
    pts = lattice_points(m)
    n_prim, n_cells = len(z), len(pts)
    sc_frac = ((frac[:, None, :] + pts[None, :, :]) @ np.linalg.inv(m.astype(np.float64))).reshape(-1, 3)
    sc_frac = sc_frac - np.floor(sc_frac)
    s2p = np.repeat(np.arange(n_prim), n_cells).astype(np.int32)
    p2s = (np.arange(n_prim) * n_cells).astype(np.int32)
    img_ptr, img_vec = minimum_images(sc_frac, p2s, m, lattice)
    return Supercell(z=np.repeat(z, n_cells), frac=sc_frac, lattice=m @ lattice, matrix=m, points=pts, s2p=s2p,
                     p2s=p2s, prim_z=z, prim_frac=frac, prim_lattice=lattice, img_ptr=img_ptr, img_vec=img_vec)


def compact_force_constants(hvp, sc: Supercell) -> np.ndarray:
    """Compact force constants ``[n_prim, N, 3, 3]`` in eV/A^2: Phi[k, j, a, b] = (H e_{p2s[k], a})[j, b], H the
    supercell Hessian.  ``hvp(v [K,N,3]) -> [K,N,3]`` computes H v for K directions; it is called once, with the
    3 n_prim unit directions on the ``p2s`` atoms."""
    n_prim, n = len(sc.p2s), len(sc.s2p)
    v = np.zeros((n_prim, 3, n, 3))
    for a in range(3):
        v[np.arange(n_prim), a, sc.p2s, a] = 1.0
    cols = np.asarray(hvp(v.reshape(3 * n_prim, n, 3)), dtype=np.float64)
    return np.ascontiguousarray(cols.reshape(n_prim, 3, n, 3).transpose(0, 2, 1, 3))


def third_order_force_constants(hvp_at, sc: Supercell, displacement: float) -> np.ndarray:
    """Compact third-order force constants ``[n_prim, N, N, 3, 3, 3]`` in eV/A^3 (phono3py's compact layout) by
    central differences of Hessians: Phi3[k, j', j'', a, b, c] = (H+ - H-)[j' b, j'' c] / 2h, H+- the supercell
    Hessian with atom ``p2s[k]`` moved by +-h (``displacement``, A) along the Cartesian axis a.  Returned as computed
    (not symmetrised).

    ``hvp_at(frac [N, 3], v [K, N, 3]) -> [K, N, 3]`` computes H v (eV/A^2) for the supercell ``sc`` with the
    fractional coordinates ``frac`` (same lattice); it is called 6 n_prim times, each with the 3N unit directions.
    ValueError unless ``displacement`` is finite and > 0."""
    h = float(displacement)
    if not (np.isfinite(h) and h > 0):
        raise ValueError(f"displacement must be finite and positive, got {displacement!r}")
    n_prim, n = len(sc.p2s), len(sc.s2p)
    inv = np.linalg.inv(np.asarray(sc.lattice, dtype=np.float64))
    cols = np.eye(3 * n).reshape(3 * n, n, 3)
    out = np.empty((n_prim, n, n, 3, 3, 3))
    for k in range(n_prim):
        for a in range(3):
            hs = []
            for sgn in (1.0, -1.0):
                frac = np.array(sc.frac, dtype=np.float64)
                frac[sc.p2s[k]] += sgn * h * inv[a]  # Cartesian step h e_a in supercell fractional coordinates
                hv = np.asarray(hvp_at(frac % 1.0, cols), dtype=np.float64).reshape(3 * n, 3 * n)  # row c: H e_c
                hs.append(hv.T)  # H[j' b, j'' c]
            d = (hs[0] - hs[1]) / (2.0 * h)
            out[k, :, :, a] = d.reshape(n, 3, n, 3).transpose(0, 2, 1, 3)
    return out


def acoustic_sum_rule(fc: np.ndarray, p2s: np.ndarray) -> tuple[np.ndarray, float]:
    """Copy of ``fc`` with the self-term correction Phi(k0, k0) -= sum_j Phi(k0, j), and the largest entry of the
    correction (eV/A^2)."""
    corr = fc.sum(axis=1)  # [n_prim, 3, 3]
    out = fc.copy()
    out[np.arange(len(p2s)), p2s] -= corr
    return out, float(np.abs(corr).max()) if corr.size else 0.0


def thermal_properties_from_frequencies(freqs, temperatures) -> dict:
    """Harmonic thermodynamics per primitive cell from the frequencies ``[Q, 3 n_prim]`` (THz) of a uniform q mesh.

    Modes with nu < 1e-3 THz are left out (acoustic modes at Gamma and imaginary modes); ``n_imaginary`` counts the
    modes below -1e-3 THz.  ``free_energy`` F = ZPE + k T sum ln(1 - e^-x) and ``zero_point_energy`` sum h nu / 2 in
    eV, ``entropy`` k sum [x / (e^x - 1) - ln(1 - e^-x)] and ``heat_capacity`` (C_v) k sum x^2 e^x / (e^x - 1)^2 in
    eV/K, with x = h nu / k T and every sum divided by Q."""
    nu = np.asarray(freqs, dtype=np.float64)
    n_q = nu.shape[0] if nu.ndim > 1 else 1
    nu = nu.reshape(-1)
    e = H_EV_PER_THZ * nu[nu >= THERMAL_CUTOFF_THZ]
    temps = np.atleast_1d(np.asarray(temperatures, dtype=np.float64))
    zpe = 0.5 * float(e.sum()) / n_q
    f, s, c = np.full(len(temps), zpe), np.zeros(len(temps)), np.zeros(len(temps))
    for i, t in enumerate(temps):
        if t <= 0:
            continue
        x = e / (KB * t)
        em = np.exp(-x)
        ln = np.log1p(-em)
        f[i] = zpe + KB * t * float(ln.sum()) / n_q
        s[i] = KB * float((x * em / -np.expm1(-x) - ln).sum()) / n_q
        c[i] = KB * float((x * x * em / np.expm1(-x) ** 2).sum()) / n_q
    return {"temperatures": temps, "free_energy": f, "entropy": s, "heat_capacity": c, "zero_point_energy": zpe,
            "n_imaginary": int((nu < -THERMAL_CUTOFF_THZ).sum())}


def gamma_mesh(mesh) -> np.ndarray:
    """[n1 n2 n3, 3] reduced q-points (i/n1, j/n2, k/n3) of a full Gamma-centred mesh."""
    mesh = np.asarray(mesh, dtype=np.int64).reshape(-1)
    if mesh.shape != (3,) or np.any(mesh < 1):
        raise ValueError(f"mesh must be three positive integers, got {mesh.tolist()}")
    axes = [np.arange(n) / n for n in mesh]
    return np.array(np.meshgrid(*axes, indexing="ij")).reshape(3, -1).T.copy()


def tetrahedra(mesh, prim_lattice, diagonal=None) -> np.ndarray:
    """[6, 4, 3] int32 corner offsets (in {0, 1}) of the 6 equal-volume tetrahedra of a cell of the Gamma-centred
    ``mesh`` that share one body diagonal of the cell: the shortest in Cartesian reciprocal space (phonopy's choice; the
    first of equal ones), or the one ``diagonal`` (0: 0 -> e1+e2+e3, 1, 2, 3: axis 1, 2, 3 reflected) names.  For the
    diagonal 0 -> e1+e2+e3 the tetrahedra are {0, e_i, e_i + e_j, e1+e2+e3} over the permutations (i, j, k)."""
    mesh = np.asarray(mesh, dtype=np.int64).reshape(3)
    g = np.linalg.inv(np.asarray(prim_lattice, dtype=np.float64)).T / mesh[:, None]  # rows: mesh steps (1/A)
    flips = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]])
    if diagonal is None:
        diagonal = int(np.argmin([np.linalg.norm((1 - 2 * f) @ g) for f in flips]))
    eye = np.eye(3, dtype=np.int64)
    tets = np.array([[np.zeros(3, np.int64), eye[i], eye[i] + eye[j], np.ones(3, np.int64)]
                     for i, j, _ in itertools.permutations(range(3))])
    f = flips[diagonal]
    return np.ascontiguousarray(np.where(f == 1, 1 - tets, tets), dtype=np.int32)


def cif_displacement_matrices(u_cart, prim_lattice) -> np.ndarray:
    """Cartesian displacement matrices ``u_cart [..., 3, 3]`` (A^2) in the CIF convention (Grosse-Kunstleve and Adams,
    as phonopy): U_cif = N^-1 A^-1 U A^-T N^-1, A = ``prim_lattice``^T (lattice vectors as columns) and
    N = diag(|a*|, |b*|, |c*|), a* the rows of inv(prim_lattice)^T.  An isotropic u I becomes u cos(a*_i, a*_j)."""
    lat = np.asarray(prim_lattice, dtype=np.float64).reshape(3, 3)
    recip = np.linalg.inv(lat).T  # rows a*, b*, c* (no 2 pi); A^-1 = recip
    m = recip / np.linalg.norm(recip, axis=1)[:, None]  # N^-1 A^-1
    return m @ np.asarray(u_cart, dtype=np.float64) @ m.T


def _signed_thz(lam: torch.Tensor) -> torch.Tensor:
    """Frequencies (THz) of the eigenvalues of D (eV/(A^2 amu)), imaginary modes negative."""
    return torch.sign(lam) * torch.sqrt(torch.abs(lam)) * THZ_PER_SQRT_EV_A2_AMU


def _temperatures(temperatures) -> np.ndarray:
    """``temperatures`` (K) as a 1-D fp64 array; ValueError unless every one is finite and >= 0."""
    temps = np.asarray(temperatures, dtype=np.float64).reshape(-1)
    if not np.all(np.isfinite(temps)) or np.any(temps < 0):
        raise ValueError(f"temperatures must be finite and non-negative, got {temps.tolist()}")
    return temps


def _zero_gamma_acoustic(nu: torch.Tensor) -> None:
    """Sets the three modes of smallest |nu| of row 0 (Gamma on a Gamma-centred mesh) to 0, in place."""
    nu[0, torch.argsort(nu[0].abs(), stable=True)[:3]] = 0.0


def _zero_gamma_rows(nu: torch.Tensor, q: np.ndarray) -> None:
    """Sets the three modes of smallest |nu| to 0, in place, in every row of ``nu`` whose reduced wave vector ``q``
    (the same rows, [Q, 3]) is Gamma: every component within 1e-9 of an integer."""
    rows = np.nonzero(np.all(np.abs(q - np.round(q)) <= 1e-9, axis=1))[0]
    if len(rows):
        r = torch.as_tensor(rows).to(nu.device)
        nu[r[:, None], torch.argsort(nu[r].abs(), dim=1, stable=True)[:, :3]] = 0.0


def _mesh_indices(mesh, q: np.ndarray) -> np.ndarray:
    """[Q] int64 indices of the reduced ``q`` [Q, 3] on the full Gamma-centred ``mesh``; ValueError unless q * mesh is
    integral to 1e-8."""
    m = np.asarray(mesh, dtype=np.int64).reshape(-1)
    x = q * m
    if not np.all(np.isfinite(x)) or np.any(np.abs(x - np.round(x)) > 1e-8):
        raise ValueError(f"qpoints must lie on the {m.tolist()} mesh (q * mesh integral), got {q.tolist()}")
    idx = np.round(x).astype(np.int64) % m
    return (idx[:, 0] * m[1] + idx[:, 1]) * m[2] + idx[:, 2]


def _degenerate_set_ids(nu: torch.Tensor) -> torch.Tensor:
    """int64 [..., 3n]: the degenerate set of each mode of nu [..., 3n] (ascending along the last axis), numbered from 0
    along that axis: adjacent modes closer than ``DEGENERACY_THZ`` share a set."""
    gap = (nu[..., 1:] - nu[..., :-1]).abs() >= DEGENERACY_THZ
    return torch.cat([torch.zeros_like(gap[..., :1], dtype=torch.long), gap.long().cumsum(-1)], -1)


def _degenerate_average(gamma: torch.Tensor, nu: torch.Tensor) -> torch.Tensor:
    """gamma [T, 3n] averaged over each set of degenerate modes of nu [3n] (``_degenerate_set_ids``), and 0 for the
    modes below ``THERMAL_CUTOFF_THZ``."""
    sid = _degenerate_set_ids(nu)
    n_sets = int(sid[-1]) + 1
    sums = torch.zeros(gamma.shape[0], n_sets, dtype=gamma.dtype, device=gamma.device).index_add_(1, sid, gamma)
    counts = torch.bincount(sid, minlength=n_sets).to(gamma.dtype)
    return torch.where(nu >= THERMAL_CUTOFF_THZ, (sums / counts)[:, sid], 0.0)


def _degenerate_operators(nu: torch.Tensor) -> torch.Tensor:
    """[N, 3n, 3n]: per row of nu [N, 3n] the matrix that averages over its degenerate sets (the grouping of
    ``_degenerate_average``), A[q, i, j] = 1 / |set| when modes i and j of q share a set, else 0 (symmetric)."""
    sid = _degenerate_set_ids(nu)
    same = (sid[:, :, None] == sid[:, None, :]).to(nu.dtype)
    return same / same.sum(-1, keepdim=True)


def _set_average(x: torch.Tensor, nu: torch.Tensor) -> torch.Tensor:
    """x [N, 3n] averaged over the degenerate sets of each row of nu [N, 3n] (``_degenerate_operators``), and 0 for the
    modes below ``THERMAL_CUTOFF_THZ``."""
    avg = (_degenerate_operators(nu) @ x[..., None])[..., 0]
    return torch.where(nu >= THERMAL_CUTOFF_THZ, avg, 0.0)


def _hat_matrix(x: torch.Tensor, grid: torch.Tensor, h: float) -> torch.Tensor:
    """[X, M]: the hat functions max(0, 1 - |x - w_k| / h) of the uniform ``grid`` w_k = k h [M] at the points ``x``
    [X]; Gamma_hat(x) = this @ Gamma_k, the piecewise-linear interpolant, 0 beyond the last hat."""
    return (1.0 - (x[:, None] - grid[None, :]).abs() / h).clamp_min(0.0)


def _hilbert_matrix(x: torch.Tensor, grid: torch.Tensor, h: float) -> torch.Tensor:
    """[X, M]: Delta(x) = this @ Gamma_k, the Hilbert transform of the odd extension of ``_hat_matrix``'s interpolant
    (DESIGN.md section 12.9), in closed form:

        Delta(x) = (1/pi) sum_{k >= 1} Gamma_k [H_k(x) + H_k(-x)],
        H_k(x) = [g(x - w_k + h) - 2 g(x - w_k) + g(x - w_k - h)] / h,   g(x) = x ln|x|,  g(0) = 0

    Column 0 (w_0 = 0, where the odd extension is 0) is 0."""
    def g(u):
        return torch.where(u == 0, 0.0, u * torch.log(torch.where(u == 0, 1.0, u.abs())))

    def hk(u):
        return (g(u + h) - 2.0 * g(u) + g(u - h)) / h

    k = (hk(x[:, None] - grid[None, :]) + hk(-x[:, None] - grid[None, :])) / math.pi
    k[:, 0] = 0.0
    return k


def _gaussian_sigma(width) -> float | None:
    """The standard deviation (THz) of a Gaussian of FWHM ``width``, width / (2 sqrt(2 ln 2)); None for None, and
    ValueError unless it is finite and > 0."""
    if width is None:
        return None
    w = float(width)
    if not (np.isfinite(w) and w > 0):
        raise ValueError(f"width must be finite and positive, got {width!r}")
    return w / (2.0 * math.sqrt(2.0 * math.log(2.0)))


def fibonacci_directions(n: int) -> np.ndarray:
    """[n, 3] unit vectors of a Fibonacci sphere: d_i = (r cos phi_i, r sin phi_i, z_i), z_i = 1 - (2 i + 1) / n,
    r = sqrt(1 - z_i^2), phi_i = i pi (3 - sqrt 5)."""
    i = np.arange(n, dtype=np.float64)
    z = 1.0 - (2.0 * i + 1.0) / n
    r = np.sqrt(1.0 - z * z)
    phi = i * (math.pi * (3.0 - math.sqrt(5.0)))
    return np.stack([r * np.cos(phi), r * np.sin(phi), z], axis=1)


def translation_table(sc: Supercell) -> np.ndarray:
    """[n_cells, N] int32 ``perm[l, j]``: the supercell atom that the lattice translation R_l (``sc.points[l]``) moves
    atom j to.  Atom j = k n_cells + l' goes to k n_cells + (the point R_l + R_l' reduced modulo the supercell lattice),
    found by integer arithmetic in primitive fractional coordinates, so any integer M works."""
    m = np.asarray(sc.matrix, dtype=np.int64)
    det = int(round(np.linalg.det(m)))
    adj = np.round(np.linalg.inv(m) * det).astype(np.int64)  # det M^-1, integral

    def code(n):  # the point n modulo the supercell lattice, as one integer
        x = (n @ adj) % det
        return (x[..., 0] * det + x[..., 1]) * det + x[..., 2]

    pts = np.asarray(sc.points, dtype=np.int64)
    n_cells = len(pts)
    keys = code(pts)
    order = np.argsort(keys)
    cell = order[np.searchsorted(keys[order], code(pts[:, None, :] + pts[None, :, :]))]  # [l, l']
    n_prim = len(sc.p2s)
    perm = (np.arange(n_prim)[None, :, None] * n_cells + cell[:, None, :]).reshape(n_cells, n_prim * n_cells)
    return np.ascontiguousarray(perm, dtype=np.int32)


def _expand_compact(x: torch.Tensor, perm_inv: torch.Tensor) -> torch.Tensor:
    """[3N, 3N] supercell matrix X_sc[(T_l(p2s k), a), (T_l(j), b)] = x[k, j, a, b] of the compact x [n_prim, N, 3, 3],
    atom-major (T_l(p2s k) = k n_cells + l); perm_inv [n_cells, N] long, perm_inv[l, perm[l, j]] = j."""
    n = x.shape[1]
    return x[:, perm_inv].reshape(n, n, 3, 3).permute(0, 2, 1, 3).reshape(3 * n, 3 * n)


def sampling_modes(phi_sc: torch.Tensor, masses: np.ndarray, temperature: float, *, quantum: bool,
                   frequency_floor: float):
    """The modes of the supercell force constants ``phi_sc`` [3N, 3N] (eV/A^2, on the device) and the sampling
    amplitudes of ``effective_force_constants`` (DESIGN.md section 12.12), for the atom ``masses`` [N] (amu).

    D_sc = phi_sc / sqrt(m m'), made symmetric as (D + D^T) / 2, is diagonalised by ``torch.linalg.eigh`` in fp64.
    Mode lam (signed THz, as ``Phonons.frequencies``) is sampled at nu~ = max(|nu|, ``frequency_floor``) with the
    amplitude A (amu^1/2 A), A^2 = C / nu~ coth(h nu~ / 2 k T) (``quantum``, C = ``DISPLACEMENT_A2_AMU_THZ``) or
    k T (``THZ_PER_SQRT_EV_A2_AMU`` / nu~)^2 (classical); the three modes of smallest |nu| (the translations) get 0.
    Returns ``(nu [3N], evecs [3N, 3N] row lam the unit mode vector, amp [3N], n_imaginary)``, ``n_imaginary`` the
    number of modes below -``THERMAL_CUTOFF_THZ``.  The displacement covariance of the samples is
    sum_lam A_lam^2 (e_lam / sqrt m)(e_lam / sqrt m)^T."""
    inv = torch.as_tensor(np.repeat(1.0 / np.sqrt(np.asarray(masses, dtype=np.float64)), 3)).to(phi_sc.device)
    d = phi_sc * inv[:, None] * inv[None, :]
    lam, e = torch.linalg.eigh(0.5 * (d + d.T))
    nu = _signed_thz(lam)
    nt = nu.abs().clamp_min(frequency_floor)
    t = float(temperature)
    if quantum:
        occ = 1.0 / torch.tanh(H_OVER_KB_K_PER_THZ * nt / (2.0 * t)) if t > 0 else torch.ones_like(nt)
        a2 = DISPLACEMENT_A2_AMU_THZ / nt * occ
    else:
        a2 = KB * t * (THZ_PER_SQRT_EV_A2_AMU / nt) ** 2
    a2[torch.argsort(nu.abs(), stable=True)[:3]] = 0.0
    return nu, e.T.contiguous(), torch.sqrt(a2), int((nu < -THERMAL_CUTOFF_THZ).sum())


def check_effective_arguments(temperature, n_atoms: int, n_cells: int, *, n_samples, n_iterations, mixing, quantum,
                              frequency_floor, seed, batch_size) -> float:
    """The temperature (K) as a float; ValueError for any argument ``effective_force_constants`` rejects."""
    t = float(temperature)
    if not (math.isfinite(t) and t >= 0):
        raise ValueError(f"temperature must be finite and non-negative, got {temperature!r}")
    if not quantum and t == 0:
        raise ValueError("a classical distribution at T = 0 has zero amplitude: use quantum=True or T > 0")
    if int(n_iterations) != n_iterations or n_iterations < 1:
        raise ValueError(f"n_iterations must be an integer >= 1, got {n_iterations!r}")
    if not (0 < float(mixing) <= 1):
        raise ValueError(f"mixing must lie in (0, 1], got {mixing!r}")
    if not (math.isfinite(float(frequency_floor)) and frequency_floor > 0):
        raise ValueError(f"frequency_floor must be finite and positive, got {frequency_floor!r}")
    if int(batch_size) != batch_size or batch_size < 1:
        raise ValueError(f"batch_size must be an integer >= 1, got {batch_size!r}")
    if int(seed) != seed or seed < 0 or seed >= 2**63:
        raise ValueError(f"seed must be an integer in [0, 2^63), got {seed!r}")
    if int(n_samples) != n_samples or n_samples * n_cells < 3 * n_atoms - 3:
        raise ValueError(f"n_samples * n_cells = {n_samples} * {n_cells} must be at least 3N - 3 = {3 * n_atoms - 3}: "
                         "fewer samples leave the fit underdetermined")
    return t


def effective_force_constants(forces, sc: Supercell, fc0, temperature, *, kernels=None, device="cuda",
                              n_samples: int = 256, n_iterations: int = 5, mixing: float = 0.5, quantum: bool = True,
                              frequency_floor: float = 0.5, seed: int = 0, batch_size: int = 16):
    """Temperature-dependent effective harmonic force constants by stochastic sampling (sTDEP / self-consistent
    phonons; DESIGN.md section 12.12).  Returns ``(fc [n_prim, N, 3, 3], info)``.

    ``forces(frac [M, N, 3] torch fp64) -> (F [M, N, 3] fp64, E [M] fp64)`` gives the forces (eV/A) and total energies
    (eV) of M copies of the supercell ``sc`` with the fractional coordinates ``frac`` (same lattice, not wrapped);
    it is called with at most ``batch_size`` copies, first once with the reference positions.  ``fc0`` are the
    starting compact force constants (``CHGNet.phonons``); the self-term acoustic-sum-rule correction of ``Phonons``
    is applied to them first.  Iteration i:

    1. the supercell modes of Phi_i and their amplitudes at ``temperature`` (K), ``quantum`` or classical
       (``sampling_modes``);
    2. ``n_samples`` displacement samples u_s = M^-1/2 sum_lam e_lam A_lam xi_s,lam with normal variates that are a
       function of (``seed``, i, s, lam) only, as fp32 fractional coordinates, u_s being the displacement those
       coordinates carry (``chg_sample_displacements``);
    3. their forces, and the moments G_c, B and S folded over the supercell translations
       (``chg_displacement_moments``), dF = F - F_0 with F_0 the forces of the reference positions;
    4. the fit Phi_fit = -B G+: G is the full Gram matrix of the displacements, projected on the complement of the
       rigid translations, and G+ inverts it by ``eigh`` treating eigenvalues <= 1e-10 max as zero.  The samples hold
       no mass-weighted translation, so the fit is undetermined along three directions; the projection fixes them by
       the acoustic sum rule (sum_j Phi[k, j] = 0), and for harmonic forces the fit is exact.  Returned as computed
       (not symmetrised); Phi_i+1 = Phi_i + ``mixing`` (Phi_fit - Phi_i).

    ``info``: ``temperature``, ``quantum``, ``harmonic_force_constants`` (``fc0``) and ``history``, one dict per
    iteration with ``max_change`` max |Phi_fit - Phi_i| (eV/A^2), ``n_imaginary`` (modes of Phi_i below
    -``THERMAL_CUTOFF_THZ`` in the supercell), ``sigma_a`` and ``u0``; and the last iteration's ``sigma_a`` and ``u0``:

    * ``sigma_a``: Knoop's anharmonicity measure of Phi_fit, sqrt(sum_s |dF_s + Phi_sc u_s|^2 / S), S = sum_s |dF_s|^2,
      from the moments (S + 2 <Phi_fit, B> + <Phi_fit, G Phi_fit>).  The sum cancels in fp64, so values below ~1e-7
      are rounding;
    * ``u0`` (eV per primitive cell): the TDEP free-energy correction < E_s - E_0 + F_0 . u_s - u_s Phi_sc u_s / 2 >
      / n_cells with Phi_fit.  F(T) ~ ``Phonons(fc, sc).thermal_properties(mesh, T)["free_energy"] + u0``.

    ``kernels`` holds ``sample_displacements`` and ``displacement_moments`` (default: the CUDA kernels on ``device``).
    ValueError for the arguments ``check_effective_arguments`` rejects."""
    n_prim, n = len(sc.p2s), len(sc.s2p)
    n_cells = len(sc.points)
    t = check_effective_arguments(temperature, n, n_cells, n_samples=n_samples, n_iterations=n_iterations,
                                  mixing=mixing, quantum=quantum, frequency_floor=frequency_floor, seed=seed,
                                  batch_size=batch_size)
    fc0 = np.asarray(fc0, dtype=np.float64)
    if fc0.shape != (n_prim, n, 3, 3):
        raise ValueError(f"force constants must have shape {[n_prim, n, 3, 3]}, got {list(fc0.shape)}")
    if kernels is None:
        from chgnet_b200._lib import CudaKernels

        kernels = CudaKernels(device)
    dev, f64 = torch.device(device), torch.float64
    perm = translation_table(sc)
    perm_inv = np.empty_like(perm)
    np.put_along_axis(perm_inv, perm, np.arange(n)[None, :].repeat(n_cells, 0), axis=1)
    perm_t = torch.as_tensor(perm).to(dev)
    perm_inv_t = torch.as_tensor(perm_inv.astype(np.int64)).to(dev)
    masses = ATOMIC_MASSES[np.asarray(sc.z) - 1]
    inv_sqrt_m = torch.as_tensor(1.0 / np.sqrt(masses)).to(dev)
    frac_ref = torch.as_tensor(np.ascontiguousarray(sc.frac, dtype=np.float64)).to(dev)
    lat = np.ascontiguousarray(sc.lattice, dtype=np.float64)
    lat_t, inv_lat_t = torch.as_tensor(lat).to(dev), torch.as_tensor(np.linalg.inv(lat)).to(dev)
    n3, n_g = 3 * n, 9 * n_prim * n
    # the rigid translations t_a[j, b] = delta_ab / sqrt N and the projector on their complement
    trans = torch.zeros(3, n3, dtype=f64, device=dev)
    for a in range(3):
        trans[a, a::3] = 1.0 / math.sqrt(n)
    proj = torch.eye(n3, dtype=f64, device=dev) - trans.T @ trans

    bs = min(int(batch_size), int(n_samples))
    frac = torch.empty(bs * n, 3, dtype=torch.float32, device=dev)
    u = torch.empty(bs, n, 3, dtype=f64, device=dev)
    f0, e0 = forces(frac_ref.to(torch.float32).to(f64).view(1, n, 3))
    f0 = f0.reshape(n, 3).to(dev, f64).contiguous()
    e0 = e0.reshape(-1)[:1].to(dev, f64)
    acc = torch.empty(2 * n_g + 2, dtype=f64, device=dev)
    energies = torch.empty(int(n_samples), dtype=f64, device=dev)
    phi = torch.as_tensor(acoustic_sum_rule(fc0, sc.p2s)[0]).to(dev)
    history = []
    for it in range(int(n_iterations)):
        _, evecs, amp, n_imag = sampling_modes(_expand_compact(phi, perm_inv_t), masses, t, quantum=quantum,
                                               frequency_floor=frequency_floor)
        acc.zero_()
        for s0 in range(0, int(n_samples), bs):
            m = min(bs, int(n_samples) - s0)
            kernels.sample_displacements(evecs, amp, inv_sqrt_m, frac_ref, lat_t, inv_lat_t, seed, it, s0,
                                         frac[: m * n], u[:m])
            f, e = forces(frac[: m * n].view(m, n, 3).to(f64))
            kernels.displacement_moments(u[:m], f.reshape(m, n, 3).to(dev, f64).contiguous(), f0, perm_t, acc)
            energies[s0 : s0 + m] = e.reshape(-1).to(dev, f64)
        g_c, b = acc[:n_g].view(n_prim * 3, n3), acc[n_g : 2 * n_g].view(n_prim * 3, n3)
        ss, wf = acc[2 * n_g], acc[2 * n_g + 1]
        g = _expand_compact(g_c.view(n_prim, 3, n, 3).permute(0, 2, 1, 3), perm_inv_t)
        gp = proj @ g @ proj
        lam, v = torch.linalg.eigh(0.5 * (gp + gp.T))
        keep = lam > 1e-10 * lam.max()
        vk = v[:, keep]
        fit_rows = -((b @ vk) / lam[keep]) @ vk.T  # [3 n_prim, 3N], rows (k, a), columns (j, b)
        fit = fit_rows.view(n_prim, 3, n, 3).permute(0, 2, 1, 3)
        res2 = ss + 2.0 * (fit_rows * b).sum() + ((fit_rows @ g) * fit_rows).sum()
        sigma = float(torch.sqrt(res2.clamp_min(0.0) / ss)) if float(ss) > 0 else 0.0
        u0 = float(((energies - e0).sum() + wf - 0.5 * (fit_rows * g_c).sum()) / (n_samples * n_cells))
        history.append({"max_change": float((fit - phi).abs().max()), "n_imaginary": n_imag, "sigma_a": sigma,
                        "u0": u0})
        phi = phi + float(mixing) * (fit - phi)
    info = {"temperature": t, "quantum": bool(quantum), "harmonic_force_constants": fc0, "history": history,
            "sigma_a": history[-1]["sigma_a"], "u0": history[-1]["u0"]}
    return np.ascontiguousarray(phi.cpu().numpy()), info


class Phonons:
    """Harmonic phonons of a crystal from its compact supercell force constants (``CHGNet.phonons``).

    Attributes: ``force_constants`` ``[n_prim, N, 3, 3]`` eV/A^2 as computed (not symmetrised), relative to
    ``supercell`` = ``(z, frac, lattice)``; ``p2s`` / ``s2p`` the atom maps (supercell atom j = k n_cells + l);
    ``asr_correction`` the largest entry of the acoustic-sum-rule correction (eV/A^2); ``masses`` of the primitive
    atoms (amu, ``chgnet_b200.dynamics.ATOMIC_MASSES``); ``force_constants3`` ``[n_prim, N, N, 3, 3, 3]`` eV/A^3 (the
    ``fc3`` argument, as computed; None without it), which ``linewidths`` and ``thermal_conductivity`` need.

    D(q) follows phonopy: the phase of the full interatomic vector r_j - r_k (basis offsets included) over the minimum
    images of the supercell, each weighted by 1 / multiplicity; built from the force constants with the self-term
    acoustic-sum-rule correction Phi(k0, k0) -= sum_j Phi(k0, j), made Hermitian as (D + D^H)/2.  ``kernels`` is the
    object whose ``dynamical_matrices`` builds D (default: the CUDA kernels on ``device``)."""

    # D(q) chunks stay below this many bytes (complex128)
    chunk_bytes = 1 << 28
    # q-points per batched eigendecomposition in dos and group_velocities (cuSOLVER rejects batches of ~30 000)
    eigh_batch = 4096
    # joint_dos and phase_space: targets per chg_joint_dos call keep its output and scratch below this many bytes
    jdos_chunk_bytes = 1 << 28
    # dynamic_structure_factor and powder_spectrum: rows per chg_broadened_spectrum call keep its scratch below this
    # many bytes (or at one group of rows, when a group alone needs more)
    sqw_chunk_bytes = 1 << 28

    # linewidths and thermal_conductivity: q1 per chg_phonon_interaction / chg_imag_self_energy call keep P, the
    # tetrahedron weights and both calls' scratch below this many bytes
    ph3_chunk_bytes = 1 << 28
    # thermal_conductivity_lbte: the collision matrices of all temperatures are built in one pass over the targets when
    # they fit in this many bytes (fp64, M^2 per temperature), else in groups of temperatures
    lbte_matrix_bytes = 8 << 30
    # spectral_function: report frequencies evaluated per pass (the interpolation and Hilbert matrices are [F, M])
    spectrum_points_per_pass = 4096
    # thermal_conductivity_wigner: q per chg_coherence_conductivity call keep dD/dQ and the call's scratch below this
    # many bytes (at least one q)
    wigner_chunk_bytes = 1 << 28
    # isotope_linewidths and the mass_variances of the conductivities: targets per chg_isotope_scattering call keep
    # its overlaps, scratch and output below this many bytes (at least one target)
    isotope_chunk_bytes = 1 << 28

    def __init__(self, force_constants: np.ndarray, sc: Supercell, *, fc3=None, device="cuda", kernels=None) -> None:
        if kernels is None:
            from chgnet_b200._lib import CudaKernels

            kernels = CudaKernels(device)
        self.kernels, self.device = kernels, torch.device(device)
        self.force_constants = np.asarray(force_constants, dtype=np.float64)
        n_prim, n = len(sc.p2s), len(sc.s2p)
        if self.force_constants.shape != (n_prim, n, 3, 3):
            raise ValueError(f"force constants must have shape {[n_prim, n, 3, 3]}, got {list(self.force_constants.shape)}")
        self.cell = sc
        self.supercell = (sc.z, sc.frac, sc.lattice)
        self.p2s, self.s2p = sc.p2s, sc.s2p
        self.masses = ATOMIC_MASSES[sc.prim_z - 1]
        fc, self.asr_correction = acoustic_sum_rule(self.force_constants, sc.p2s)
        dev = self.device
        self._fc = torch.as_tensor(fc).to(dev)
        self._img_ptr = torch.as_tensor(sc.img_ptr).to(dev)
        self._img_vec = torch.as_tensor(sc.img_vec).to(dev)
        self._s2p = torch.as_tensor(sc.s2p).to(dev)
        self._inv_sqrt_m = torch.as_tensor(1.0 / np.sqrt(self.masses)).to(dev)
        self._lattice = torch.as_tensor(np.ascontiguousarray(sc.prim_lattice, dtype=np.float64)).to(dev)
        self.force_constants3 = None
        if fc3 is not None:
            self.force_constants3 = np.asarray(fc3, dtype=np.float64)
            if self.force_constants3.shape != (n_prim, n, n, 3, 3, 3):
                raise ValueError(f"third-order force constants must have shape {[n_prim, n, n, 3, 3, 3]}, got "
                                 f"{list(self.force_constants3.shape)}")
            self._fc3 = torch.as_tensor(np.ascontiguousarray(self.force_constants3)).to(dev)

    def dynamical_matrices(self, qpoints) -> torch.Tensor:
        """D(q) ``[Q, 3 n_prim, 3 n_prim]`` complex128 on the device, in eV/(A^2 amu), for reduced ``qpoints [Q,3]``."""
        q = torch.as_tensor(np.ascontiguousarray(np.asarray(qpoints, dtype=np.float64).reshape(-1, 3))).to(self.device)
        n3 = 3 * len(self.p2s)
        d = torch.empty(q.shape[0], n3, n3, dtype=torch.complex128, device=self.device)
        self.kernels.dynamical_matrices(self._fc, self._img_ptr, self._img_vec, self._s2p, self._inv_sqrt_m, q, d)
        return d

    def _eigh_chunks(self, q, *, eigenvectors: bool, matrices_per_q: int = 1, eigh_batch=math.inf):
        """Yields ``(slice, nu, e or None)`` per chunk of ``q``: frequencies (THz) and eigenvectors of D on the device,
        at most ``eigh_batch`` q keeping ``matrices_per_q`` complex128 [3n, 3n] per q below ``chunk_bytes``."""
        n3 = 3 * len(self.p2s)
        chunk = max(1, min(self.chunk_bytes // (matrices_per_q * 16 * n3 * n3), eigh_batch))
        for s in range(0, len(q), chunk):
            d = self.dynamical_matrices(q[s : s + chunk])
            lam, e = torch.linalg.eigh(d) if eigenvectors else (torch.linalg.eigvalsh(d), None)
            yield slice(s, s + chunk), _signed_thz(lam), e

    def frequencies(self, qpoints, *, eigenvectors: bool = False):
        """Frequencies ``[Q, 3 n_prim]`` in THz at the reduced ``qpoints`` (``[Q,3]`` or ``[3]``), ascending per q;
        an imaginary mode (negative eigenvalue of D) is given as a negative number, nu = sign(lambda) sqrt|lambda|
        x 15.633304 THz.  With ``eigenvectors``, also ``[Q, 3 n_prim, 3 n_prim]`` complex128 whose column m is the unit
        eigenvector of mode m (phonopy's layout and phase convention).  D is built and diagonalised on the device in
        chunks of q that keep it below ``chunk_bytes``.  The force constants should come from a relaxed structure:
        otherwise the modes describe the curvature at a non-stationary point, and unstable modes appear as imaginary
        frequencies rather than being hidden."""
        q = np.asarray(qpoints, dtype=np.float64)
        single = q.ndim == 1
        q = q.reshape(-1, 3)
        n3 = 3 * len(self.p2s)
        freqs = np.empty((len(q), n3))
        vecs = np.empty((len(q), n3, n3), dtype=np.complex128) if eigenvectors else None
        for s, nu, e in self._eigh_chunks(q, eigenvectors=eigenvectors):
            freqs[s] = nu.cpu().numpy()
            if eigenvectors:
                vecs[s] = e.cpu().numpy()
        if single:
            freqs = freqs[0]
            vecs = None if vecs is None else vecs[0]
        return (freqs, vecs) if eigenvectors else freqs

    def thermal_properties(self, mesh, temperatures) -> dict:
        """Harmonic thermodynamics per primitive cell on a full Gamma-centred ``mesh`` (n1, n2, n3) at ``temperatures``
        (K): ``free_energy`` and ``zero_point_energy`` in eV, ``entropy`` and ``heat_capacity`` (C_v) in eV/K, and
        ``n_imaginary``, the number of modes below -1e-3 THz over the mesh.  Modes with nu < 1e-3 THz are left out of
        the sums (``thermal_properties_from_frequencies``)."""
        return thermal_properties_from_frequencies(self.frequencies(gamma_mesh(mesh)), temperatures)

    def group_velocities(self, qpoints) -> np.ndarray:
        """Group velocities ``[Q, 3 n_prim, 3]`` (``[3 n_prim, 3]`` for one q) in THz*A (100 m/s) at the reduced
        ``qpoints``: the Cartesian d nu / dQ = d omega / dk of each mode, in the order of ``frequencies(qpoints)``.

        For a non-degenerate mode, v_c = c^2 Re<e|dD/dQ_c|e> / (2 |nu|) with c = ``THZ_PER_SQRT_EV_A2_AMU``: the
        derivative of the signed frequency, so an imaginary mode (nu < 0) gets the derivative of -c sqrt|lambda|.  In a
        set of degenerate modes (adjacent |d nu| < ``DEGENERACY_THZ``) component c comes from the ascending eigenvalues
        of E^H dD/dQ_c E restricted to the set (phonopy's convention); the set's sum does not depend on the basis.
        Modes with |nu| < ``THERMAL_CUTOFF_THZ`` get 0.  D, dD/dQ (``chg_dynamical_matrix_derivatives``) and the
        eigenvectors are computed on the device in chunks of q that keep them below ``chunk_bytes``."""
        q = np.asarray(qpoints, dtype=np.float64)
        single = q.ndim == 1
        q = np.ascontiguousarray(q.reshape(-1, 3))
        n3 = 3 * len(self.p2s)
        dev, c2 = self.device, THZ_PER_SQRT_EV_A2_AMU**2
        out = np.empty((len(q), n3, 3))
        # D and its three derivatives per q
        for s, nu, e in self._eigh_chunks(q, eigenvectors=True, matrices_per_q=4, eigh_batch=self.eigh_batch):
            qd = torch.as_tensor(q[s]).to(dev)
            nq = qd.shape[0]
            dd = torch.empty(nq, 3, n3, n3, dtype=torch.complex128, device=dev)
            self.kernels.dynamical_matrix_derivatives(self._fc, self._img_ptr, self._img_vec, self._s2p,
                                                      self._inv_sqrt_m, qd, self._lattice, dd)
            m = e.conj().transpose(1, 2)[:, None] @ dd @ e[:, None]  # [nq, 3, n3, n3]
            dlam = torch.diagonal(m, dim1=-2, dim2=-1).real.clone()  # [nq, 3, n3]
            # degenerate sets: set ids ascending along the (ascending) modes
            sid = _degenerate_set_ids(nu)
            idx = torch.nonzero((sid[:, 1:] == sid[:, :-1]).any(dim=1)).flatten()
            if idx.numel():
                ids = sid[idx]
                mb = m[idx] * (ids[:, :, None] == ids[:, None, :])[:, None]  # block diagonal, one block per set
                # shift set k by k * delta, delta > twice the Gershgorin radius: the ascending eigenvalues of the
                # shifted matrix come set by set, each set's own eigenvalues in ascending order
                delta = 2.5 * mb.abs().sum(-1).amax(-1) + torch.finfo(torch.float64).tiny  # [K, 3]
                shift = ids[:, None, :] * delta[:, :, None]
                ev = torch.linalg.eigvalsh(mb + torch.diag_embed(shift.to(torch.complex128)))
                dlam[idx] = ev - shift
            anu = nu.abs()[:, None, :]
            v = torch.where(anu >= THERMAL_CUTOFF_THZ, c2 * dlam / (2 * anu.clamp_min(THERMAL_CUTOFF_THZ)), 0.0)
            out[s] = v.transpose(1, 2).cpu().numpy()
        return out[0] if single else out

    def _mesh_frequencies(self, mesh, *, projected: bool = False):
        """Frequencies ``[N, 3 n_prim]`` (THz, ascending per q) on the device at the points of the full Gamma-centred
        ``mesh``, and with ``projected`` the eigenvector weights ``[N, 3 n_prim, n_prim]`` sum_a |e_(k a)|^2 (else
        None): D(q) and ``torch.linalg.eigvalsh`` (``eigh``) in chunks of at most ``eigh_batch`` q that keep D below
        ``chunk_bytes``."""
        q = gamma_mesh(mesh)
        n_prim = len(self.p2s)
        n3, dev = 3 * n_prim, self.device
        nu = torch.empty(len(q), n3, dtype=torch.float64, device=dev)
        proj = torch.empty(len(q), n3, n_prim, dtype=torch.float64, device=dev) if projected else None
        for s, nu_s, e in self._eigh_chunks(q, eigenvectors=projected, eigh_batch=self.eigh_batch):
            if projected:
                proj[s] = (e.abs() ** 2).view(-1, n_prim, 3, n3).sum(dim=2).transpose(1, 2)
            nu[s] = nu_s
        return nu, proj

    def dos(self, mesh, frequency_points=None, *, projected: bool = False) -> dict:
        """Phonon density of states by the linear tetrahedron method on a full Gamma-centred ``mesh`` (n1, n2, n3).

        Returns ``frequency_points`` (THz; default 201 points from the lowest to the highest frequency of the mesh,
        imaginary modes as negative numbers), ``total_dos`` (states/THz per primitive cell, integrating to 3 n_prim),
        ``integrated_dos`` and, with ``projected``, ``projected_dos`` [n_prim, F]: the DOS projected on each primitive
        atom with the weights sum_a |e_(k a)|^2 of the eigenvectors (the projections add up to ``total_dos``).

        Each mesh cell is cut into 6 tetrahedra around its shortest body diagonal (``tetrahedra``), and each band,
        ascending per q, is interpolated on its own (phonopy's method; its known error at band crossings falls with
        the mesh).  Frequencies, eigenvector weights and the DOS (``chg_tetrahedron_dos``) stay on the device until
        the result is returned."""
        mesh = tuple(int(n) for n in np.asarray(mesh).reshape(-1))
        n_prim, dev = len(self.p2s), self.device
        nu, proj = self._mesh_frequencies(mesh, projected=projected)
        if frequency_points is None:
            t = torch.arange(201, dtype=torch.float64, device=dev) / 200  # lerp ends exactly on the maximum
            omega = torch.lerp(nu.min().expand(201), nu.max().expand(201), t)
        else:
            omega = torch.as_tensor(np.asarray(frequency_points, dtype=np.float64).reshape(-1)).to(dev)
        tets = torch.as_tensor(tetrahedra(mesh, self.cell.prim_lattice)).to(dev)
        total, integrated = torch.empty_like(omega), torch.empty_like(omega)
        pdos = torch.empty(n_prim, len(omega), dtype=torch.float64, device=dev) if projected else None
        self.kernels.tetrahedron_dos(nu, mesh, tets, omega, total, integrated, proj, pdos)
        out = {"frequency_points": omega.cpu().numpy(), "total_dos": total.cpu().numpy(),
               "integrated_dos": integrated.cpu().numpy()}
        if projected:
            out["projected_dos"] = pdos.cpu().numpy()
        return out

    def thermal_displacement_matrices(self, mesh, temperatures) -> dict:
        """Anisotropic thermal displacement matrices of the primitive atoms on a full Gamma-centred ``mesh`` (n1, n2,
        n3) at ``temperatures`` (K, finite and >= 0, else ValueError):

            U_k(T) = hbar / (2 m_k N_q) sum_q sum_nu [1 + 2 n(nu, T)] / omega_nu(q) Re[e_k,nu(q) e_k,nu(q)^H]

        over the N_q points of the mesh (Gamma included, phonopy's normalisation), e_k the 3-component block of atom k
        in the unit eigenvector, omega = 2 pi nu and 1 + 2n = 1 + 2 / expm1(h nu / k T) (1 at T = 0).  Modes with
        nu < ``THERMAL_CUTOFF_THZ`` are left out (imaginary and near-zero modes, as in ``thermal_properties``), and so
        are, whatever their value, the three modes of smallest |nu| at Gamma: a Gamma acoustic mode lifted above the
        cutoff by force-constant noise would otherwise add ~2 k T / (h nu^2) each.  The sum over the full mesh is
        real (q and -q pair up), so only Re(e e^H) is accumulated.

        Returns ``temperatures`` [T], ``cartesian`` [T, n_prim, 3, 3] and ``cif`` [T, n_prim, 3, 3] in A^2
        (``cif_displacement_matrices``), and ``n_imaginary``, the number of modes below -``THERMAL_CUTOFF_THZ`` over
        the mesh, as in ``thermal_properties``: U is not meaningful when it is not 0.  D(q), the eigenvectors and the
        sums (``chg_thermal_displacements``) stay on the device, in chunks of at most ``eigh_batch`` q; only the
        [T, n_prim, 6] sums are copied back."""
        temps = _temperatures(temperatures)
        q = gamma_mesh(mesh)
        n_prim, dev = len(self.p2s), self.device
        t = torch.as_tensor(temps).to(dev)
        acc = torch.zeros(len(temps), n_prim, 6, dtype=torch.float64, device=dev)
        n_imaginary = torch.zeros((), dtype=torch.int64, device=dev)
        for s, nu, e in self._eigh_chunks(q, eigenvectors=True, eigh_batch=self.eigh_batch):
            n_imaginary += (nu < -THERMAL_CUTOFF_THZ).sum()
            if s.start == 0:  # q index 0 is Gamma
                _zero_gamma_acoustic(nu)
            # eigh returns column-major matrices: e.mT is the mode-major layout of the kernel, without a copy
            self.kernels.thermal_displacements(nu, e.mT.contiguous(), t, THERMAL_CUTOFF_THZ, acc)
        v = acc.cpu().numpy() * (DISPLACEMENT_A2_AMU_THZ / len(q)) / self.masses[None, :, None]
        cart = v[..., [[0, 5, 4], [5, 1, 3], [4, 3, 2]]]  # Voigt xx, yy, zz, yz, xz, xy -> 3x3
        return {"temperatures": temps, "cartesian": cart, "cif": cif_displacement_matrices(cart, self.cell.prim_lattice),
                "n_imaginary": int(n_imaginary)}

    def _jdos_mesh(self, mesh, temperatures):
        """The mesh, its frequencies on the device with the three modes of smallest |nu| at Gamma set to 0 (still
        ascending), ``n_imaginary`` (counted before that), the tetrahedra and the temperatures (None or [T] on the
        device) for ``joint_dos`` and ``phase_space``."""
        temps = None if temperatures is None else _temperatures(temperatures)
        mesh = tuple(int(n) for n in np.asarray(mesh).reshape(-1))
        nu = self._mesh_frequencies(mesh)[0]
        n_imaginary = (nu < -THERMAL_CUTOFF_THZ).sum()
        _zero_gamma_acoustic(nu)
        tets = torch.as_tensor(tetrahedra(mesh, self.cell.prim_lattice)).to(self.device)
        t = None if temps is None else torch.as_tensor(temps).to(self.device)
        return mesh, nu, n_imaginary, tets, temps, t

    def _joint_dos_chunks(self, mesh, nu, tets, targets, omega, t) -> torch.Tensor:
        """[Q, 1 + T, 2, F] from ``chg_joint_dos`` over chunks of targets whose output and scratch stay below
        ``jdos_chunk_bytes``."""
        n_slots = 1 + (0 if t is None else len(t))
        per_target = 8 * (JDOS_MAX_CHUNKS + 1) * n_slots * 2 * omega.shape[1]
        chunk = max(1, self.jdos_chunk_bytes // per_target)
        out = torch.empty(len(targets), n_slots, 2, omega.shape[1], dtype=torch.float64, device=self.device)
        for s in range(0, len(targets), chunk):
            self.kernels.joint_dos(nu, mesh, tets, targets[s : s + chunk], omega[s : s + chunk], t,
                                   THERMAL_CUTOFF_THZ, out[s : s + chunk])
        return out

    def joint_dos(self, mesh, qpoints, frequency_points=None, temperatures=None) -> dict:
        """Two-phonon joint densities of states (phono3py's ``--jdos``) at ``qpoints`` ([Q, 3] or [3], reduced, on the
        full Gamma-centred ``mesh``: q * mesh integral to 1e-8, else ValueError), in 1/THz:

            D2(1)(q, w) = 1/N sum [d(w + nu1 - nu2) + d(w - nu1 + nu2)]   (class 1: absorption)
            D2(2)(q, w) = 1/N sum d(w - nu1 - nu2)                        (class 2: decay)
            N2(1)(q, w; T) = 1/N sum (n1 - n2) [d(w + nu1 - nu2) - d(w - nu1 + nu2)]
            N2(2)(q, w; T) = 1/N sum (n1 + n2 + 1) d(w - nu1 - nu2)

        over the N mesh points q1 and every ordered band pair, nu1 = nu_l1(q1), nu2 = nu_l2(q - q1) and
        n = 1 / expm1(h nu / k T) (0 at T = 0).  The deltas are integrated over q1 by the linear tetrahedron method
        with the tetrahedra of ``dos``.  A corner where nu1 or nu2 is below ``THERMAL_CUTOFF_THZ`` is left out
        (imaginary and near-zero modes), and so are the three modes of smallest |nu| at Gamma, whatever their value:
        n ~ k T / h nu diverges for an acoustic mode that force-constant noise lifts above the cutoff.

        Returns ``frequency_points`` [F] (THz; default 201 points from 0 to twice the highest frequency of the mesh),
        ``jdos`` [Q, 2, F] (classes 1 and 2), ``n_imaginary`` (the modes below -``THERMAL_CUTOFF_THZ`` over the
        mesh, as in ``thermal_properties``) and, with ``temperatures`` (K, finite and >= 0, else ValueError),
        ``temperatures`` and ``weighted_jdos`` [T, Q, 2, F].  Frequencies and sums (``chg_joint_dos``) stay on the
        device until the result is returned."""
        q = np.asarray(qpoints, dtype=np.float64)
        single = q.ndim == 1
        q = q.reshape(-1, 3)
        idx = _mesh_indices(mesh, q)
        mesh, nu, n_imaginary, tets, temps, t = self._jdos_mesh(mesh, temperatures)
        targets = torch.as_tensor(idx.astype(np.int32)).to(self.device)
        if frequency_points is None:
            top = 2 * nu.max()
            omega = torch.lerp(torch.zeros_like(top).expand(201), top.expand(201),
                               torch.arange(201, dtype=torch.float64, device=self.device) / 200)
        else:
            omega = torch.as_tensor(np.asarray(frequency_points, dtype=np.float64).reshape(-1)).to(self.device)
        out = self._joint_dos_chunks(mesh, nu, tets, targets, omega[None].expand(len(q), -1).contiguous(), t)
        res = {"frequency_points": omega.cpu().numpy(), "jdos": out[:, 0].cpu().numpy(),
               "n_imaginary": int(n_imaginary)}
        if temps is not None:
            res["temperatures"] = temps
            res["weighted_jdos"] = out[:, 1:].transpose(0, 1).cpu().numpy()
        if single:
            res["jdos"] = res["jdos"][0]
            if temps is not None:
                res["weighted_jdos"] = res["weighted_jdos"][:, 0]
        return res

    def phase_space(self, mesh, temperatures=None) -> dict:
        """The three-phonon phase space: the quantities of ``joint_dos`` per mode, at w = nu_l(q) for every q of the
        full Gamma-centred ``mesh`` (n1, n2, n3) and every mode l.

        Returns ``frequencies`` [N, 3 n_prim] (THz, the mesh frequencies the sums use: the three modes of smallest |nu|
        at Gamma set to 0), ``jdos`` [N, 3 n_prim, 2] (classes 1 and 2, 1/THz), ``average_jdos`` [2] (the mean over
        the modes kept, nu >= ``THERMAL_CUTOFF_THZ``; the screening proxy for anharmonic scattering: a small phase space
        means weak three-phonon scattering) and ``n_imaginary``; with ``temperatures`` also ``temperatures``,
        ``weighted_jdos`` [T, N, 3 n_prim, 2] and ``average_weighted_jdos`` [T, 2].  Modes below the cutoff get 0.
        Every q is a target of ``chg_joint_dos``, in chunks of ``jdos_chunk_bytes``; everything stays on the device
        until the result is returned."""
        mesh, nu, n_imaginary, tets, temps, t = self._jdos_mesh(mesh, temperatures)
        targets = torch.arange(nu.shape[0], dtype=torch.int32, device=self.device)
        out = self._joint_dos_chunks(mesh, nu, tets, targets, nu, t)  # [N, 1 + T, 2, 3n]
        kept = nu >= THERMAL_CUTOFF_THZ
        out = torch.where(kept[:, None, None, :], out, 0.0).permute(1, 0, 3, 2)  # [1 + T, N, 3n, 2]
        n_kept = kept.sum().clamp_min(1)
        avg = out.sum(dim=(1, 2)) / n_kept  # [1 + T, 2]
        res = {"frequencies": nu.cpu().numpy(), "jdos": out[0].cpu().numpy(), "average_jdos": avg[0].cpu().numpy(),
               "n_imaginary": int(n_imaginary)}
        if temps is not None:
            res["temperatures"] = temps
            res["weighted_jdos"] = out[1:].cpu().numpy()
            res["average_weighted_jdos"] = avg[1:].cpu().numpy()
        return res

    def _scattering_coefficients(self, scattering_lengths) -> np.ndarray:
        """[n_prim] b_k / sqrt(m_k) from the mapping {atomic number: coherent scattering length}; ValueError if a
        species of the primitive cell is missing or its length is not finite."""
        coef = np.empty(len(self.p2s))
        for k, z in enumerate(self.cell.prim_z):
            b = scattering_lengths.get(int(z)) if hasattr(scattering_lengths, "get") else None
            if b is None or not np.isfinite(float(b)):
                raise ValueError(f"scattering_lengths needs a finite coherent scattering length for atomic number "
                                 f"{int(z)}, got {b!r}")
            coef[k] = float(b) / math.sqrt(self.masses[k])
        return coef

    def _debye_waller(self, debye_waller_mesh, temps):
        """U [T, n_prim, 6] (Voigt, A^2) on the device from ``thermal_displacement_matrices`` on ``debye_waller_mesh``
        and that call's ``n_imaginary``, or (None, None) for no Debye-Waller factor."""
        if debye_waller_mesh is None:
            return None, None
        td = self.thermal_displacement_matrices(debye_waller_mesh, temps)
        u = td["cartesian"][..., [0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1]]
        return torch.as_tensor(np.ascontiguousarray(u)).to(self.device), td["n_imaginary"]

    def _structure_factor_chunks(self, q_red, g, u, t, coef):
        """Yields ``(slice, nu, weights, n_imaginary)`` per eigh chunk of the rows (scattering vectors Q = q_red + g):
        the frequencies at q_red (THz, the three modes of smallest |nu| set to 0 where q_red is Gamma), the
        ``chg_structure_factors`` output [T, rows, 3n, 2] and the chunk's modes below -``THERMAL_CUTOFF_THZ`` (counted
        before the Gamma rule), all on the device.  ``g`` [Q, 3] is any integer vector: |F| does not depend on it."""
        dev = self.device
        n3 = 3 * len(self.p2s)
        q_red = np.ascontiguousarray(q_red, dtype=np.float64)
        g = np.ascontiguousarray(g, dtype=np.float64)
        kcart = 2 * math.pi * (q_red + g) @ np.linalg.inv(self.cell.prim_lattice).T
        frac = torch.as_tensor(np.ascontiguousarray(self.cell.prim_frac, dtype=np.float64)).to(dev)
        coef = torch.as_tensor(coef).to(dev)
        for s, nu, e in self._eigh_chunks(q_red, eigenvectors=True, eigh_batch=self.eigh_batch):
            n_imaginary = (nu < -THERMAL_CUTOFF_THZ).sum()
            _zero_gamma_rows(nu, q_red[s])
            out = torch.empty(len(t), nu.shape[0], n3, 2, dtype=torch.float64, device=dev)
            # eigh returns column-major matrices: e.mT is the mode-major layout of the kernel, without a copy
            self.kernels.structure_factors(nu, e.mT.contiguous(), torch.as_tensor(kcart[s]).to(dev),
                                           torch.as_tensor(g[s]).to(dev), frac, coef, u, t, THERMAL_CUTOFF_THZ, out)
            yield s, nu, out, n_imaginary

    def _broaden(self, nu, w, row0, group_size, omega, sigma, out) -> None:
        """``chg_broadened_spectrum`` of the rows [row0, row0 + len(nu)) of nu [R, 3n] and w [T, R, 3n, 2] into out
        [T, n_groups, F], in calls of as many rows as keep the call's scratch (``sqw_scratch_doubles``) within
        ``sqw_chunk_bytes``: whole groups where two fit (a call may straddle one group more than it holds), else a
        part of a group, at least one row (whose scratch, one [T, F] map, is the least a call can have)."""
        n_rows, n3 = nu.shape
        n_t, n_f = w.shape[0], omega.shape[0]
        per_group = 8 * sqw_scratch_doubles(min(group_size, n_rows), n3, n_t, 0, group_size, n_f)
        n_fit = self.sqw_chunk_bytes // per_group
        if n_fit >= 2:
            rows = (n_fit - 1) * group_size
        else:  # r < group_size rows over two groups take ceil(r 3n / 32) chunks of 2 T F doubles
            rows = max(1, min(group_size, self.sqw_chunk_bytes // (16 * n_t * n_f) * 32 // n3))
        for a in range(0, n_rows, rows):
            b = min(a + rows, n_rows)
            self.kernels.broadened_spectrum(nu[a:b], w[:, a:b].contiguous(), row0 + a, group_size, omega, sigma, out)

    def dynamic_structure_factor(self, qpoints, temperatures, scattering_lengths, *, debye_waller_mesh=None,
                                 frequency_points=None, width=None) -> dict:
        """Coherent one-phonon neutron scattering S(Q, omega) per mode at the scattering vectors ``qpoints`` ([Q, 3]
        or [3], reduced in the primitive reciprocal basis; the result drops the Q axis for one [3] vector):

            F_nu(Q, T) = sum_k b_k m_k^-1/2 exp(-W_k) (K . e_k,nu(q)) exp(-2 pi i G . x_k),  W_k = K^T U_k(T) K / 2
            S+_nu = C (n + 1) / nu |F_nu|^2  (energy loss, omega = +nu),  S-_nu = C n / nu |F_nu|^2  (gain, -nu)

        with K = 2 pi Q inv(prim_lattice)^T the Cartesian scattering vector (1/A, 2 pi included), G = floor(Q + 1/2),
        q = Q - G, e_k,nu(q) atom k's block of the eigenvector of ``frequencies`` (phonopy's phase convention), x_k
        the fractional positions, m_k in amu, n = 1 / expm1(h nu / k T) (0 at T = 0) and C = h / (8 pi^2 amu THz)
        (``DISPLACEMENT_A2_AMU_THZ``).  The phase exp(-2 pi i G . x_k) makes |F| independent of the G that reduces Q.
        ``scattering_lengths`` maps every atomic number of the primitive cell to its coherent scattering length b
        (finite, else ValueError); S is in units of b^2 per primitive cell, e.g. fm^2 for b in fm (fcc Cu:
        ``{29: 7.718}``).  U_k(T) is ``thermal_displacement_matrices(debye_waller_mesh, temperatures)``, or W = 0
        without ``debye_waller_mesh``.  Modes with nu < ``THERMAL_CUTOFF_THZ`` get S = 0, and where q is Gamma so do
        the three modes of smallest |nu| (the Bragg peak is elastic).

        Returns ``qpoints`` (q = Q - G), ``frequencies`` [Q, 3n] (THz, with those Gamma modes set to 0), ``stokes``
        (S+) and ``anti_stokes`` (S-) [T, Q, 3n], ``temperatures`` and ``n_imaginary`` (the modes below
        -``THERMAL_CUTOFF_THZ`` over the Q evaluated); with ``debye_waller_mesh`` also ``debye_waller_n_imaginary``;
        with ``frequency_points`` (THz, may be negative; needs ``width``) also ``spectrum`` [T, Q, F]
        = sum_nu [S+ g(omega - nu) + S- g(omega + nu)] in b^2/THz per primitive cell, g the normalised Gaussian of
        FWHM ``width`` (THz) cut at 8 sigma.  Non-finite Q, bad temperatures, width <= 0 and missing species raise
        ValueError.  D(q), the eigenvectors and the structure factors (``chg_structure_factors``, then
        ``chg_broadened_spectrum``) stay on the device in chunks of at most ``eigh_batch`` q."""
        big_q = np.asarray(qpoints, dtype=np.float64)
        single = big_q.ndim == 1
        big_q = big_q.reshape(-1, 3)
        if not np.all(np.isfinite(big_q)):
            raise ValueError(f"qpoints must be finite, got {big_q.tolist()}")
        temps = _temperatures(temperatures)
        if frequency_points is not None and width is None:
            raise ValueError("frequency_points needs a width (THz)")
        sigma = _gaussian_sigma(width)
        coef = self._scattering_coefficients(scattering_lengths)
        u, dw_imag = self._debye_waller(debye_waller_mesh, temps)
        g = np.floor(big_q + 0.5)
        q = big_q - g
        dev, n3 = self.device, 3 * len(self.p2s)
        t = torch.as_tensor(temps).to(dev)
        nu_all = torch.empty(len(q), n3, dtype=torch.float64, device=dev)
        sqw = torch.empty(len(temps), len(q), n3, 2, dtype=torch.float64, device=dev)
        spec = omega = None
        if frequency_points is not None:
            omega = torch.as_tensor(np.asarray(frequency_points, dtype=np.float64).reshape(-1)).to(dev)
            spec = torch.zeros(len(temps), len(q), len(omega), dtype=torch.float64, device=dev)
        n_imaginary = torch.zeros((), dtype=torch.int64, device=dev)
        for s, nu, w, n_im in self._structure_factor_chunks(q, g, u, t, coef):
            n_imaginary += n_im
            nu_all[s], sqw[:, s] = nu, w
            if spec is not None:
                self._broaden(nu, w, s.start, 1, omega, sigma, spec)
        res = {"qpoints": q, "frequencies": nu_all.cpu().numpy(), "stokes": sqw[..., 0].cpu().numpy(),
               "anti_stokes": sqw[..., 1].cpu().numpy(), "temperatures": temps, "n_imaginary": int(n_imaginary)}
        if dw_imag is not None:
            res["debye_waller_n_imaginary"] = dw_imag
        if spec is not None:
            res["frequency_points"] = omega.cpu().numpy()
            res["spectrum"] = spec.cpu().numpy()
        if single:
            res["qpoints"], res["frequencies"] = res["qpoints"][0], res["frequencies"][0]
            for key in ("stokes", "anti_stokes", "spectrum"):
                if key in res:
                    res[key] = res[key][:, 0]
        return res

    def powder_spectrum(self, q_magnitudes, frequency_points, temperatures, scattering_lengths, *, width,
                        n_directions=500, debye_waller_mesh=None) -> dict:
        """Powder-averaged coherent one-phonon spectrum S(|Q|, omega) in b^2/THz per primitive cell: the spectrum of
        ``dynamic_structure_factor`` averaged over the ``n_directions`` unit vectors d_i of ``fibonacci_directions``
        (a plain mean), K = |Q| d_i in the Cartesian frame of the lattice as given, Q = K prim_lattice^T / 2 pi.

        ``q_magnitudes`` [M] in 1/A (2 pi included; finite and >= 0), ``frequency_points`` [F] in THz (may be
        negative), ``width`` the FWHM of the Gaussian (THz, > 0), ``n_directions`` >= 1; the other arguments as in
        ``dynamic_structure_factor``, and the same errors.  Returns ``q_magnitudes``, ``frequency_points``,
        ``temperatures``, ``spectrum`` [T, M, F] and ``n_imaginary`` (over all M n_directions vectors); with
        ``debye_waller_mesh`` also ``debye_waller_n_imaginary``.  The M n_directions rows run as contiguous groups of
        ``n_directions`` through the eigh chunks; frequencies, eigenvectors and weights stay on the device, and
        ``chg_broadened_spectrum`` adds each chunk's rows to their shells, so only [T, M, F] is copied back."""
        qm = np.asarray(q_magnitudes, dtype=np.float64).reshape(-1)
        if not np.all(np.isfinite(qm)) or np.any(qm < 0):
            raise ValueError(f"q_magnitudes must be finite and non-negative, got {qm.tolist()}")
        n_dir = int(n_directions)
        if n_dir != n_directions or n_dir < 1:
            raise ValueError(f"n_directions must be a positive integer, got {n_directions!r}")
        temps = _temperatures(temperatures)
        if width is None:
            raise ValueError("powder_spectrum needs a width (THz)")
        sigma = _gaussian_sigma(width)
        coef = self._scattering_coefficients(scattering_lengths)
        u, dw_imag = self._debye_waller(debye_waller_mesh, temps)
        kcart = (qm[:, None, None] * fibonacci_directions(n_dir)[None]).reshape(-1, 3)
        big_q = kcart @ np.asarray(self.cell.prim_lattice, dtype=np.float64).T / (2 * math.pi)
        g = np.floor(big_q + 0.5)
        dev = self.device
        t = torch.as_tensor(temps).to(dev)
        omega = torch.as_tensor(np.asarray(frequency_points, dtype=np.float64).reshape(-1)).to(dev)
        spec = torch.zeros(len(temps), len(qm), len(omega), dtype=torch.float64, device=dev)
        n_imaginary = torch.zeros((), dtype=torch.int64, device=dev)
        for s, nu, w, n_im in self._structure_factor_chunks(big_q - g, g, u, t, coef):
            n_imaginary += n_im
            self._broaden(nu, w, s.start, n_dir, omega, sigma, spec)
        res = {"q_magnitudes": qm, "frequency_points": omega.cpu().numpy(), "temperatures": temps,
               "spectrum": spec.cpu().numpy(), "n_imaginary": int(n_imaginary)}
        if dw_imag is not None:
            res["debye_waller_n_imaginary"] = dw_imag
        return res

    def _three_phonon_mesh(self, mesh, temperatures):
        """The mesh, its frequencies [N, 3n] on the device with the three modes of smallest |nu| at Gamma set to 0,
        the mode-major eigenvectors [N, mode, 3n], ``n_imaginary`` (counted before that), the tetrahedra and the
        temperatures (fp64 array; None allowed) for the three-phonon methods.  ValueError without fc3."""
        if self.force_constants3 is None:
            raise ValueError("this needs third-order force constants: build the phonons with "
                             "CHGNet.phonons(..., third_order=True), or pass fc3 to Phonons")
        temps = None if temperatures is None else _temperatures(temperatures)
        return (*self._mesh_modes(mesh), temps)

    def _mesh_modes(self, mesh):
        """The mesh, its frequencies [N, 3n] on the device with the three modes of smallest |nu| at Gamma set to 0, the
        mode-major eigenvectors [N, mode, 3n], ``n_imaginary`` (counted before that) and the tetrahedra: one
        eigendecomposition of the mesh in chunks of at most ``eigh_batch`` q."""
        mesh = tuple(int(n) for n in np.asarray(mesh).reshape(-1))
        q = gamma_mesh(mesh)
        n3, dev = 3 * len(self.p2s), self.device
        nu = torch.empty(len(q), n3, dtype=torch.float64, device=dev)
        e = torch.empty(len(q), n3, n3, dtype=torch.complex128, device=dev)
        for s, nu_s, e_s in self._eigh_chunks(q, eigenvectors=True, eigh_batch=self.eigh_batch):
            nu[s] = nu_s
            e[s] = e_s.mT  # eigh's columns are the modes: the kernels read them mode-major
        n_imaginary = int((nu < -THERMAL_CUTOFF_THZ).sum())
        _zero_gamma_acoustic(nu)
        tets = torch.as_tensor(tetrahedra(mesh, self.cell.prim_lattice)).to(dev)
        return mesh, nu, e, n_imaginary, tets

    def _q1_chunk(self, n_t) -> int:
        """q1 per ``chg_phonon_interaction`` / ``chg_imag_self_energy`` call: P, both calls' scratch within
        ``ph3_chunk_bytes`` (at least one)."""
        n_prim = len(self.p2s)
        nb = 3 * n_prim
        per_q1 = 8 * (nb**3 + ph3_scratch_doubles(1, n_prim, len(self.s2p)) + ise_scratch_doubles(1, nb, 0))
        fixed = 8 * ise_scratch_doubles(0, nb, n_t)
        # chg_collision_rows' scratch, collision_scratch_doubles(1, nb) = 3 nb^3 per q1, is less than the
        # chg_phonon_interaction scratch counted here and is allocated after that has been released, so this chunk
        # also bounds thermal_conductivity_lbte (and stays the chunk of thermal_conductivity, whose Gamma it shares)
        return int(max(1, min(65535, (self.ph3_chunk_bytes - fixed) // per_q1)))

    def _interaction_chunks(self, mesh, nu, e, target: int, chunk: int):
        """Yields ``(q1, P)`` per chunk of ``chunk`` q1 of the mesh, in mesh order: the mesh indices (int32, device) and
        their interaction strengths with the mesh index ``target``."""
        n_mesh = nu.shape[0]
        for s in range(0, n_mesh, chunk):
            q1 = torch.arange(s, min(s + chunk, n_mesh), dtype=torch.int32, device=self.device)
            yield q1, self._interactions(mesh, nu, e, target, q1)

    def _interactions(self, mesh, nu, e, target: int, q1: torch.Tensor) -> torch.Tensor:
        """P [len(q1), 3n, 3n, 3n] (eV^2) of the mesh index ``target`` with the mesh indices ``q1`` (int32, device)."""
        nb = 3 * len(self.p2s)
        frac = torch.as_tensor(np.ascontiguousarray(self.cell.prim_frac, dtype=np.float64)).to(self.device)
        p = torch.empty(len(q1), nb, nb, nb, dtype=torch.float64, device=self.device)
        self.kernels.phonon_interaction(self._fc3, self._img_ptr, self._img_vec, self._s2p, self._inv_sqrt_m, frac,
                                        mesh, nu, e, int(target), q1, THERMAL_CUTOFF_THZ, p)
        return p

    def _target_linewidths(self, mesh, nu, e, tets, t, target: int) -> torch.Tensor:
        """Gamma [T, 3n] (THz) of the modes of the mesh index ``target``: P and its contribution to Gamma per chunk of
        q1 (``_q1_chunk``, chunks in mesh order), then averaged over degenerate sets."""
        gamma = torch.zeros(len(t), nu.shape[1], dtype=torch.float64, device=self.device)
        omega = nu[target].contiguous()
        for q1, p in self._interaction_chunks(mesh, nu, e, target, self._q1_chunk(len(t))):
            self.kernels.imag_self_energy(nu, mesh, tets, int(target), omega, q1, p, t, THERMAL_CUTOFF_THZ, gamma)
        return _degenerate_average(gamma, omega)

    def _interaction_strength(self, mesh, q, q1=None) -> np.ndarray:
        """The interaction strengths P [Q1, 3n, 3n, 3n] (eV^2, ``chg_phonon_interaction``) of the mesh point ``q`` [3]
        with the mesh points ``q1`` [Q1, 3] (default: the whole mesh, in mesh order), q2 = q - q1 on the mesh."""
        mesh_t, nu, e, _, _, _ = self._three_phonon_mesh(mesh, None)
        target = int(_mesh_indices(mesh_t, np.asarray(q, dtype=np.float64).reshape(1, 3))[0])
        if q1 is None:
            idx = np.arange(nu.shape[0])
        else:
            idx = _mesh_indices(mesh_t, np.asarray(q1, dtype=np.float64).reshape(-1, 3))
        q1_t = torch.as_tensor(idx.astype(np.int32)).to(self.device)
        return self._interactions(mesh_t, nu, e, target, q1_t).cpu().numpy()

    def linewidths(self, mesh, qpoints, temperatures) -> dict:
        """Three-phonon linewidths (phono3py's imaginary self-energy at omega = nu, half width) of the modes at
        ``qpoints`` ([Q, 3] or [3], reduced, on the full Gamma-centred ``mesh``: q * mesh integral to 1e-8, else
        ValueError) at ``temperatures`` (K, finite and >= 0, else ValueError), in THz (DESIGN.md section 12.7):

            Gamma_l(q; T) = 18 pi / h^2 sum_{q1 l1 l2} P_l,l1,l2(q; q1) {(1 + n1 + n2) g2 + (n1 - n2) [g1+ - g1-]}

        over the N mesh points q1, q2 = q - q1 on the mesh, P the interaction strengths (eV^2, 1/N included) of the
        third-order force constants, n = 1 / expm1(h nu / k T) and g2, g1+, g1- the linear-tetrahedron weights of
        vertex q1 for d(w - nu1 - nu2), d(w + nu1 - nu2) and d(w - nu1 + nu2) with the tetrahedra of ``joint_dos``.
        Modes below ``THERMAL_CUTOFF_THZ``, and the three modes of smallest |nu| at Gamma, take no part (P = 0) and get
        0; Gamma is averaged over each set of degenerate modes at q (adjacent |d nu| < ``DEGENERACY_THZ``).  The
        lifetime is tau = 1 / (4 pi Gamma) ps.

        Returns ``frequencies`` [Q, 3n] (THz, with that Gamma rule), ``temperatures``, ``linewidths`` [T, Q, 3n] and
        ``n_imaginary`` (the modes below -``THERMAL_CUTOFF_THZ`` over the mesh).  Needs ``force_constants3``
        (``CHGNet.phonons(..., third_order=True)``), else ValueError.  Frequencies and eigenvectors of the mesh come
        from one eigendecomposition per call; P (``chg_phonon_interaction``) is made and consumed
        (``chg_imag_self_energy``) per chunk of q1 within ``ph3_chunk_bytes``, on the device."""
        q = np.asarray(qpoints, dtype=np.float64)
        single = q.ndim == 1
        q = q.reshape(-1, 3)
        idx = _mesh_indices(mesh, q)
        if temperatures is None:
            raise ValueError("linewidths needs temperatures")
        mesh, nu, e, n_imaginary, tets, temps = self._three_phonon_mesh(mesh, temperatures)
        t = torch.as_tensor(temps).to(self.device)
        gamma = torch.stack([self._target_linewidths(mesh, nu, e, tets, t, int(i)) for i in idx], 1)
        res = {"frequencies": nu[torch.as_tensor(idx).to(self.device)].cpu().numpy(), "temperatures": temps,
               "linewidths": gamma.cpu().numpy(), "n_imaginary": n_imaginary}
        if single:
            res["frequencies"], res["linewidths"] = res["frequencies"][0], res["linewidths"][:, 0]
        return res

    def _mass_variances(self, mass_variances) -> torch.Tensor:
        """``mass_variances`` as [n_prim] fp64 on the device; ValueError unless they are n_prim finite values >= 0."""
        n_prim = len(self.p2s)
        g = np.asarray(mass_variances, dtype=np.float64).reshape(-1)
        if g.shape != (n_prim,) or not np.all(np.isfinite(g)) or np.any(g < 0):
            raise ValueError(f"mass_variances must be {n_prim} finite values >= 0 (one per primitive atom), got "
                             f"{np.asarray(mass_variances).tolist()}")
        return torch.as_tensor(g).to(self.device)

    def _isotope_targets(self, mesh, nu, e, tets, g, idx) -> torch.Tensor:
        """Gamma^iso [Q, 3n] (THz) of the mesh indices ``idx`` [Q] at their own frequencies, averaged over the
        degenerate sets of each: ``chg_isotope_scattering`` per chunk of targets within ``isotope_chunk_bytes``."""
        n_mesh, nb = nu.shape
        per_target = 8 * (isotope_scratch_doubles(1, n_mesh, nb) + nb)
        chunk = int(max(1, min(65535, self.isotope_chunk_bytes // per_target)))
        targets = torch.as_tensor(np.asarray(idx, dtype=np.int32)).to(self.device)
        omega = nu[targets.long()].contiguous()
        gamma = torch.empty_like(omega)
        for s in range(0, len(targets), chunk):
            self.kernels.isotope_scattering(nu, mesh, tets, e, g, targets[s : s + chunk], omega[s : s + chunk],
                                            THERMAL_CUTOFF_THZ, gamma[s : s + chunk])
        return _set_average(gamma, omega)

    def isotope_linewidths(self, mesh, qpoints, mass_variances) -> dict:
        """Isotope (mass-disorder) scattering rates of Tamura (PRB 27, 858 (1983)), half width in THz, of the modes at
        ``qpoints`` ([Q, 3] or [3], reduced, on the full Gamma-centred ``mesh``: q * mesh integral to 1e-8, else
        ValueError), DESIGN.md section 12.11:

            Gamma^iso_l(q) = (pi / 4) nu_l^2 (1/N) sum_{q' l'} W_l'(q'; nu_l) sum_k g_k |sum_a conj(e_ka(q l)) e_ka(q' l')|^2

        with W the linear-tetrahedron vertex weight of d(nu - nu_l'(q')) (the tetrahedra of ``dos``) and g_k =
        sum_i f_i (1 - m_i / m_k)^2 the ``mass_variances`` of the primitive atoms (phono3py's ``--mass_variances``;
        n_prim finite values >= 0, else ValueError).  Vertex modes below ``THERMAL_CUTOFF_THZ`` take no part; modes
        below it, and the three modes of smallest |nu| at Gamma, get 0; Gamma^iso is averaged over each set of
        degenerate modes at q (adjacent |d nu| < ``DEGENERACY_THZ``) and does not depend on temperature.  Harmonic:
        no third-order force constants are needed.

        Returns ``frequencies`` [Q, 3n] (THz, with that Gamma rule), ``isotope_linewidths`` [Q, 3n] and
        ``n_imaginary`` (the modes below -``THERMAL_CUTOFF_THZ`` over the mesh); a single q drops the Q axis.  The
        mesh is diagonalised once per call, and the sums (``chg_isotope_scattering``) run on the device per chunk of
        targets within ``isotope_chunk_bytes``."""
        q = np.asarray(qpoints, dtype=np.float64)
        single = q.ndim == 1
        q = q.reshape(-1, 3)
        idx = _mesh_indices(mesh, q)
        g = self._mass_variances(mass_variances)
        mesh, nu, e, n_imaginary, tets = self._mesh_modes(mesh)
        gamma = self._isotope_targets(mesh, nu, e, tets, g, idx)
        res = {"frequencies": nu[torch.as_tensor(idx).to(self.device)].cpu().numpy(),
               "isotope_linewidths": gamma.cpu().numpy(), "n_imaginary": n_imaginary}
        if single:
            res["frequencies"], res["isotope_linewidths"] = res["frequencies"][0], res["isotope_linewidths"][0]
        return res

    def _extra_scattering(self, mesh, nu, e, tets, mass_variances, boundary_mfp):
        """The checked options of the conductivities: (Gamma^iso [N, 3n] of every mesh point or None, L or None)."""
        g = None if mass_variances is None else self._mass_variances(mass_variances)
        if boundary_mfp is not None:
            boundary_mfp = float(boundary_mfp)
            if not (math.isfinite(boundary_mfp) and boundary_mfp > 0):
                raise ValueError(f"boundary_mfp must be finite and positive (micrometres), got {boundary_mfp!r}")
        iso = None if g is None else self._isotope_targets(mesh, nu, e, tets, g, np.arange(nu.shape[0]))
        return iso, boundary_mfp

    def _spectrum_q1_chunk(self, n_t, n_freq) -> int:
        """q1 per ``chg_phonon_interaction`` / ``chg_self_energy_spectrum`` call in ``spectral_function``: P, the
        interaction's scratch and the spectrum's partial sums within ``ph3_chunk_bytes`` (at least one)."""
        n_prim = len(self.p2s)
        nb = 3 * n_prim
        per_q1 = 8 * (nb**3 + ph3_scratch_doubles(1, n_prim, len(self.s2p)))
        fixed = 8 * (se_scratch_doubles(nb, n_freq, n_t) + n_t * nb * n_freq)
        return int(max(1, min(65535, (self.ph3_chunk_bytes - fixed) // per_q1)))

    def _target_self_energy(self, mesh, nu, e, tets, t, target: int, grid: torch.Tensor) -> torch.Tensor:
        """Gamma [T, 3n, M] (THz) of the modes of the mesh index ``target`` at the points ``grid`` [M]: P and its
        contribution per chunk of q1 (``_spectrum_q1_chunk``, chunks in mesh order), then averaged over the degenerate
        sets of each point (``_degenerate_average``)."""
        nb, m = nu.shape[1], grid.shape[0]
        gamma = torch.zeros(len(t), nb, m, dtype=torch.float64, device=self.device)
        for q1, p in self._interaction_chunks(mesh, nu, e, target, self._spectrum_q1_chunk(len(t), m)):
            self.kernels.self_energy_spectrum(nu, mesh, tets, int(target), grid, q1, p, t, THERMAL_CUTOFF_THZ, gamma)
        avg = _degenerate_average(gamma.transpose(1, 2).reshape(-1, nb), nu[target])
        return avg.reshape(len(t), m, nb).transpose(1, 2)

    def spectral_function(self, mesh, qpoints, temperatures, frequency_points=None, *, self_energy_points=201) -> dict:
        """Frequency-resolved three-phonon self-energies and anharmonic phonon spectral functions of the modes at
        ``qpoints`` ([Q, 3] or [3], reduced, on the full Gamma-centred ``mesh``) at ``temperatures`` (K), DESIGN.md
        section 12.9.  Gamma_l(q; w) is ``linewidths``' sum with the tetrahedron weights at w instead of at nu_l, on
        the grid w_k = k h, k = 0 ... M - 1, h = 2 nu_max / (M - 1) (M = ``self_energy_points``, nu_max the highest
        mesh frequency); between the points it is the piecewise-linear interpolant, 0 beyond.  The real part is the
        exact Hilbert transform of the odd extension of that interpolant, in closed form,

            Delta_l(w) = (1/pi) PV int_0^inf Gamma_l(w') [1 / (w - w') - 1 / (w + w')] dw'

        so Sigma = Delta - i Gamma is causal, and the spectral function (1/THz) with the harmonic nu_l is

            A_l(q; w) = (1/pi) 4 nu_l^2 Gamma_l(w) / [(w^2 - nu_l^2 - 2 nu_l Delta_l(w))^2 + 4 nu_l^2 Gamma_l(w)^2]

        (0 where Gamma_l(w) = 0), which keeps int_0^inf w A dw = nu_l when it has no undamped pole.  Gamma is
        averaged over each set of degenerate modes at q at every grid point (so are Delta, A and the shifts); modes
        below ``THERMAL_CUTOFF_THZ``, and the three modes of smallest |nu| at Gamma, get 0 throughout.

        Returns ``frequencies`` [Q, 3n] (THz, with that Gamma rule), ``temperatures``, ``self_energy_points`` [M]
        (THz), ``gamma`` and ``delta`` [T, Q, 3n, M] (THz) on them, ``frequency_points`` [F] (THz; default 2 001
        points from 0 to 2 nu_max), ``spectral_function`` [T, Q, 3n, F], ``frequency_shifts`` [T, Q, 3n] = Delta_l
        (nu_l) (THz) and ``n_imaginary`` (the modes below -``THERMAL_CUTOFF_THZ`` over the mesh).  A single q drops
        the Q axis.  ValueError without ``force_constants3``, for bad temperatures, q off the mesh,
        ``self_energy_points`` not an integer >= 3, and ``frequency_points`` that are not a non-empty list of finite
        numbers >= 0.  The mesh is diagonalised once per call; P (``chg_phonon_interaction``) is made and consumed
        (``chg_self_energy_spectrum``) per chunk of q1 within ``ph3_chunk_bytes``, on the device."""
        q = np.asarray(qpoints, dtype=np.float64)
        single = q.ndim == 1
        q = q.reshape(-1, 3)
        idx = _mesh_indices(mesh, q)
        if temperatures is None:
            raise ValueError("spectral_function needs temperatures")
        if isinstance(self_energy_points, (bool, np.bool_)) or not isinstance(self_energy_points, (int, np.integer)) \
                or self_energy_points < 3:
            raise ValueError(f"self_energy_points must be an integer >= 3, got {self_energy_points!r}")
        m = int(self_energy_points)
        report = None
        if frequency_points is not None:
            report = np.asarray(frequency_points, dtype=np.float64).reshape(-1)
            if report.size == 0 or not np.all(np.isfinite(report)) or np.any(report < 0):
                raise ValueError("frequency_points must be a non-empty list of finite frequencies >= 0 (THz), got "
                                 f"{np.asarray(frequency_points).tolist()}")
        mesh, nu, e, n_imaginary, tets, temps = self._three_phonon_mesh(mesh, temperatures)
        dev, f64 = self.device, torch.float64
        t = torch.as_tensor(temps).to(dev)
        top = float(2 * nu.max())
        h = top / (m - 1)
        grid = torch.arange(m, dtype=f64, device=dev) * h
        if report is None:
            omega = torch.lerp(torch.zeros((), dtype=f64, device=dev).expand(2001),
                               torch.full((), top, dtype=f64, device=dev).expand(2001),
                               torch.arange(2001, dtype=f64, device=dev) / 2000)
        else:
            omega = torch.as_tensor(report).to(dev)
        gamma = torch.stack([self._target_self_energy(mesh, nu, e, tets, t, int(i), grid) for i in idx], 1)
        nq = nu[torch.as_tensor(idx).to(dev)]  # [Q, 3n]
        delta = gamma @ _hilbert_matrix(grid, grid, h).T  # [T, Q, 3n, M]
        shifts = (gamma * _hilbert_matrix(nq.reshape(-1), grid, h).view(*nq.shape, m)[None]).sum(-1)
        v = nq[None, :, :, None]
        a = torch.empty(*gamma.shape[:3], len(omega), dtype=f64, device=dev)
        for s in range(0, len(omega), self.spectrum_points_per_pass):  # keeps the [F, M] matrices small
            w = omega[s : s + self.spectrum_points_per_pass]
            g_rep = gamma @ _hat_matrix(w, grid, h).T  # [T, Q, 3n, F]
            d_rep = gamma @ _hilbert_matrix(w, grid, h).T
            den = (w * w - v * v - 2 * v * d_rep) ** 2 + 4 * v * v * g_rep * g_rep
            a[..., s : s + len(w)] = torch.where(
                g_rep != 0, 4 * v * v * g_rep / (math.pi * torch.where(g_rep != 0, den, 1.0)), 0.0)
        res = {"frequencies": nq.cpu().numpy(), "temperatures": temps, "self_energy_points": grid.cpu().numpy(),
               "gamma": gamma.cpu().numpy(), "delta": delta.cpu().numpy(), "frequency_points": omega.cpu().numpy(),
               "spectral_function": a.cpu().numpy(), "frequency_shifts": shifts.cpu().numpy(),
               "n_imaginary": n_imaginary}
        if single:
            res["frequencies"] = res["frequencies"][0]
            for k in ("gamma", "delta", "spectral_function", "frequency_shifts"):
                res[k] = res[k][:, 0]
        return res

    def thermal_conductivity(self, mesh, temperatures, *, mass_variances=None, boundary_mfp=None) -> dict:
        """Lattice thermal conductivity in the relaxation-time approximation on the full Gamma-centred ``mesh``, every
        mesh point a target (no symmetry reduction), in W/(m K):

            kappa(T) = 1 / (N V0) sum_{q l} C_l v_l (x) v_l tau_l,   C = k_B x^2 e^x / (e^x - 1)^2,  x = h nu / k T

        with tau = 1 / (4 pi Gamma) from ``linewidths``, v from ``group_velocities`` and V0 the primitive-cell volume.
        Modes below ``THERMAL_CUTOFF_THZ`` (and the three modes of smallest |nu| at Gamma) are left out, and so are
        modes with Gamma <= 0, whose lifetime is undefined; ``n_zero_linewidth`` [T] counts those.

        Isotope and boundary scattering (DESIGN.md section 12.11) add to Gamma by Matthiessen's rule: with
        ``mass_variances`` (g per primitive atom, as ``isotope_linewidths``) Gamma^iso, with ``boundary_mfp`` (L, in
        micrometres) Gamma^bnd = |v| / (4 pi 10^4 L), averaged over degenerate sets.  tau, the kept modes and
        ``n_zero_linewidth`` then use Gamma + Gamma^iso + Gamma^bnd.

        Returns ``temperatures``, ``kappa`` [T, 3, 3], per mode ``frequencies`` [N, 3n] (THz), ``linewidths``
        [T, N, 3n] (THz, three-phonon), ``group_velocities`` [N, 3n, 3] (THz A) and ``heat_capacity`` [T, N, 3n]
        (eV/K), and ``n_imaginary`` and ``n_zero_linewidth``; with the options also ``isotope_linewidths`` and
        ``boundary_linewidths`` [N, 3n] (THz).  Needs ``force_constants3``, else ValueError; bad temperatures,
        ``mass_variances`` that are not n_prim finite values >= 0 and a ``boundary_mfp`` that is not finite and > 0
        raise ValueError."""
        if temperatures is None:
            raise ValueError("thermal_conductivity needs temperatures")
        mesh, nu, e, n_imaginary, tets, temps = self._three_phonon_mesh(mesh, temperatures)
        iso, mfp = self._extra_scattering(mesh, nu, e, tets, mass_variances, boundary_mfp)
        dev = self.device
        t = torch.as_tensor(temps).to(dev)
        gamma = torch.stack([self._target_linewidths(mesh, nu, e, tets, t, i) for i in range(nu.shape[0])], 1)
        return self._rta_conductivity(mesh, nu, gamma, t, temps, n_imaginary, iso, mfp)[0]

    def _rta_conductivity(self, mesh, nu, gamma, t, temps, n_imaginary, iso=None, boundary_mfp=None):
        """(``thermal_conductivity``'s result, the total linewidths [T, N, 3n] on the device) from the mesh frequencies
        nu [N, 3n], the three-phonon linewidths gamma [T, N, 3n] at the temperatures t (device) and temps (array), and
        the isotope linewidths iso [N, 3n] and boundary mean free path (um) when given."""
        v = torch.as_tensor(self.group_velocities(gamma_mesh(mesh))).to(self.device)  # [N, 3n, 3]
        extra = {}
        if iso is not None:
            extra["isotope_linewidths"] = iso
        if boundary_mfp is not None:
            speed = torch.where(nu >= THERMAL_CUTOFF_THZ, torch.linalg.vector_norm(v, dim=-1), 0.0)
            extra["boundary_linewidths"] = _set_average(speed / (4 * math.pi * 1e4 * boundary_mfp), nu)
        total = gamma
        for x in extra.values():
            total = total + x[None]
        kept = nu >= THERMAL_CUTOFF_THZ
        tt = t[:, None, None]
        x = H_OVER_KB_K_PER_THZ * torch.where(kept, nu, 1.0)[None] / torch.where(tt > 0, tt, 1.0)
        em = torch.exp(-x)
        cv = torch.where(kept[None] & (tt > 0), KB * x * x * em / torch.expm1(-x) ** 2, 0.0)  # [T, N, 3n]
        use = kept[None] & (total > 0)
        tau = torch.where(use, 1.0 / (4 * math.pi * torch.where(use, total, 1.0)), 0.0)
        vv = v[:, :, :, None] * v[:, :, None, :]  # [N, 3n, 3, 3]
        vol = abs(float(np.linalg.det(self.cell.prim_lattice)))
        kappa = torch.einsum("tqm,qmab->tab", cv * tau, vv) * (KAPPA_W_PER_MK / (nu.shape[0] * vol))
        res = {"temperatures": temps, "kappa": kappa.cpu().numpy(), "frequencies": nu.cpu().numpy(),
               "linewidths": gamma.cpu().numpy(), "group_velocities": v.cpu().numpy(),
               "heat_capacity": cv.cpu().numpy(), "n_imaginary": n_imaginary,
               "n_zero_linewidth": (kept[None] & ~(total > 0)).sum(dim=(1, 2)).cpu().numpy()}
        res.update({k: x.cpu().numpy() for k, x in extra.items()})
        return res, total

    def thermal_conductivity_wigner(self, mesh, temperatures, *, mass_variances=None, boundary_mfp=None) -> dict:
        """Lattice thermal conductivity with the Wigner coherence term (Simoncelli, Marzari and Mauri, Nat. Phys. 15,
        809 (2019)) on the full Gamma-centred ``mesh``, every mesh point a target, in W/(m K) (DESIGN.md section
        12.10): kappa = kappa_P + kappa_C, kappa_P ``thermal_conductivity``'s kappa (bitwise: the same linewidths and
        the same sum) and

            kappa_C(T) = 1 / (N V0) sum_q sum_{s != s'} (nu_s + nu_s') / 4 (C_s / nu_s + C_s' / nu_s')
                         Re(V_s,s' (x) V_s',s) (Gamma_s + Gamma_s') / (2 pi [(nu_s - nu_s')^2 + (Gamma_s + Gamma_s')^2])

        with V_s,s' = c^2 <e_s| dD/dQ |e_s'> / (|nu_s| + |nu_s'|) the velocity operator (THz A, c =
        ``THZ_PER_SQRT_EV_A2_AMU``; its diagonal is the group velocity of a non-degenerate mode), C and Gamma the heat
        capacities and degenerate-averaged linewidths of ``thermal_conductivity`` (with ``mass_variances`` and
        ``boundary_mfp`` as there, Gamma is the total of section 12.11 in the Lorentzians).  The pairs are the ordered pairs of
        modes that ``thermal_conductivity`` keeps (nu >= ``THERMAL_CUTOFF_THZ``, not the three acoustic modes at Gamma,
        Gamma > 0) and that lie in different degenerate sets (adjacent |d nu| < ``DEGENERACY_THZ``): a pair inside a
        set depends on the basis eigh picks in it, and the set's basis-invariant part is already in kappa_P.

        Returns everything ``thermal_conductivity`` returns with the same options, with ``kappa`` = kappa_P + kappa_C,
        plus ``kappa_p`` and ``kappa_c`` [T, 3, 3].  Needs ``force_constants3``, else ValueError; bad temperatures and
        options raise ValueError as in ``thermal_conductivity``.  dD/dQ
        (``chg_dynamical_matrix_derivatives``) and the pair sum (``chg_coherence_conductivity``) run on the device per
        chunk of q within ``wigner_chunk_bytes``."""
        if temperatures is None:
            raise ValueError("thermal_conductivity_wigner needs temperatures")
        mesh, nu, e, n_imaginary, tets, temps = self._three_phonon_mesh(mesh, temperatures)
        iso, mfp = self._extra_scattering(mesh, nu, e, tets, mass_variances, boundary_mfp)
        dev = self.device
        t = torch.as_tensor(temps).to(dev)
        gamma = torch.stack([self._target_linewidths(mesh, nu, e, tets, t, i) for i in range(nu.shape[0])], 1)
        res, gamma = self._rta_conductivity(mesh, nu, gamma, t, temps, n_imaginary, iso, mfp)
        cv = torch.as_tensor(res["heat_capacity"]).to(dev)
        sid = _degenerate_set_ids(nu).to(torch.int32)
        q = gamma_mesh(mesh)
        n_mesh, nb = nu.shape
        per_q = 16 * 3 * nb * nb + 8 * coherence_scratch_doubles(1, nb, 0)
        chunk = int(max(1, min(65535, (self.wigner_chunk_bytes - 8 * coherence_scratch_doubles(0, nb, len(temps)))
                               // per_q)))
        kappa_c = torch.zeros(len(temps), 3, 3, dtype=torch.float64, device=dev)
        for s in range(0, n_mesh, chunk):
            sl = slice(s, s + chunk)
            qd = torch.as_tensor(q[sl]).to(dev)
            dd = torch.empty(qd.shape[0], 3, nb, nb, dtype=torch.complex128, device=dev)
            self.kernels.dynamical_matrix_derivatives(self._fc, self._img_ptr, self._img_vec, self._s2p,
                                                      self._inv_sqrt_m, qd, self._lattice, dd)
            self.kernels.coherence_conductivity(nu[sl], e[sl], dd, sid[sl], cv[:, sl].contiguous(),
                                                gamma[:, sl].contiguous(), THERMAL_CUTOFF_THZ, kappa_c)
        vol = abs(float(np.linalg.det(self.cell.prim_lattice)))
        res["kappa_p"] = res["kappa"]
        res["kappa_c"] = (kappa_c * (KAPPA_W_PER_MK / (n_mesh * vol))).cpu().numpy()
        res["kappa"] = res["kappa_p"] + res["kappa_c"]
        return res

    def _collision_passes(self, mesh, nu, e, tets, t, groups):
        """One pass over the targets per group of temperature indices in ``groups`` (P remade per pass).  Yields
        ``(group, target, gamma, rows)``: gamma [T, 3n] the degenerate-averaged linewidths of the target at all the
        temperatures t, from the first pass only (None after; made exactly as ``thermal_conductivity`` makes them), and
        rows [len(group), 3n, N, 3n] the target's rows of S, row l against column (c, l'), before any averaging:

            S[q l][c l'] = R_A[c] + R_B[-c] + R_C[q - c] + R_D[q + c]   (R by vertex q1, ``chg_collision_rows``)"""
        n_mesh, nb = nu.shape
        dev = self.device
        size = np.array(mesh)
        coords = np.stack(np.unravel_index(np.arange(n_mesh), mesh), 1)
        flat = lambda c: torch.as_tensor(np.ravel_multi_index(tuple((c % size).T), mesh)).to(dev)  # noqa: E731
        neg = flat(-coords)
        chunk = self._q1_chunk(len(t))
        for gi, group in enumerate(groups):
            tg = t[torch.as_tensor(group, dtype=torch.long).to(dev)].contiguous()
            r = torch.zeros(4, len(group), nb, n_mesh, nb, dtype=torch.float64, device=dev)
            for target in range(n_mesh):
                gamma = torch.zeros(len(t), nb, dtype=torch.float64, device=dev) if gi == 0 else None
                omega = nu[target].contiguous()
                for q1, p in self._interaction_chunks(mesh, nu, e, target, chunk):
                    if gamma is not None:
                        self.kernels.imag_self_energy(nu, mesh, tets, target, omega, q1, p, t, THERMAL_CUTOFF_THZ, gamma)
                    if len(group):
                        self.kernels.collision_rows(nu, mesh, tets, target, omega, q1, p, tg, THERMAL_CUTOFF_THZ, r)
                rows = r[0] + r[1][:, :, neg] + r[2][:, :, flat(coords[target] - coords)]
                rows = rows + r[3][:, :, flat(coords[target] + coords)]
                yield group, target, (None if gamma is None else _degenerate_average(gamma, omega)), rows

    def _collision_matrix(self, mesh, temperatures):
        """For the tests: S [T, N 3n, N 3n] (1/ps) before degenerate averaging and symmetrisation, rows and columns in
        mesh-major (q, l) order, the degenerate-averaged linewidths [T, N, 3n] (THz) and the kept mask [T, N 3n] of
        ``thermal_conductivity_lbte`` (nu >= the cutoff, the Gamma rule and Gamma > 0)."""
        mesh, nu, e, _, tets, temps = self._three_phonon_mesh(mesh, temperatures)
        n_mesh, nb = nu.shape
        t = torch.as_tensor(temps).to(self.device)
        s = torch.zeros(len(temps), n_mesh * nb, n_mesh * nb, dtype=torch.float64, device=self.device)
        gamma = torch.zeros(len(temps), n_mesh, nb, dtype=torch.float64, device=self.device)
        for _, target, g, rows in self._collision_passes(mesh, nu, e, tets, t, [list(range(len(temps)))]):
            s[:, target * nb : (target + 1) * nb] = rows.reshape(len(temps), nb, -1)
            gamma[:, target] = g
        kept = (nu >= THERMAL_CUTOFF_THZ)[None] & (gamma > 0)
        return s, gamma, kept.reshape(len(temps), -1)

    def thermal_conductivity_lbte(self, mesh, temperatures, *, pinv_cutoff=1e-8, mass_variances=None,
                                  boundary_mfp=None) -> dict:
        """Lattice thermal conductivity (W/(m K)) from the direct solution of the linearised phonon Boltzmann equation
        (Chaput, PRL 110, 265506 (2013)) on the full Gamma-centred ``mesh``, every mesh point a target (DESIGN.md
        section 12.8).  The collision matrix, symmetrised and in 1/ps,

            Omega = diag(4 pi Gamma) + S,   S[q l][c] = sum over the processes of mode q l with mode c of
                    u_q u_c 2 pi 18 pi / h^2 P g / sinh(h nu_o / 2 k T)

        (g the tetrahedron weight of the process, o its third mode, u = +1 for the mode alone on its side of the
        process, -1 for the other two), averaged over degenerate sets (rows, then columns) and made symmetric, keeps
        the modes ``thermal_conductivity`` keeps (nu >= ``THERMAL_CUTOFF_THZ``, not the three acoustic modes at Gamma,
        Gamma > 0).  With Omega = U diag(eta) U^T and X = sqrt(C) v per mode,

            kappa = 1 / (N V0) sum over eta_k > pinv_cutoff of (U^T X)_k (x) (U^T X)_k / eta_k

        which is ``thermal_conductivity``'s kappa when S = 0.  Eigenvalues <= ``pinv_cutoff`` (1/ps; the energy mode
        near 0 and small negative ones) are left out and counted.  At T = 0 kappa is 0 and no matrix is built.  With
        ``mass_variances`` and ``boundary_mfp`` (as ``thermal_conductivity``) Gamma is the total of DESIGN.md section
        12.11 on the diagonal and in the kept modes; S keeps the three-phonon processes only (as phono3py, the
        off-diagonal part of elastic isotope scattering is left out).

        Returns ``temperatures``, ``kappa`` and ``kappa_rta`` [T, 3, 3] (the latter bitwise ``thermal_conductivity``'s
        kappa with the same options), per mode ``frequencies``, ``linewidths``, ``group_velocities`` and ``heat_capacity`` as
        ``thermal_conductivity`` (and its ``isotope_linewidths`` and ``boundary_linewidths`` with the options),
        ``n_imaginary``, ``n_zero_linewidth``, ``n_dropped`` [T] (eigenvalues <=
        pinv_cutoff) and ``min_eigenvalue`` [T] (1/ps, NaN where no matrix was built).  The matrices of all
        temperatures above 0 are built in one pass over the targets when n_t M^2 8 bytes fit in ``lbte_matrix_bytes``
        (M: the modes at or above the cutoff), else in groups of temperatures with P remade per group; ValueError
        with the bytes needed when one temperature alone does not fit.  Needs ``force_constants3``, else ValueError;
        bad temperatures and a ``pinv_cutoff`` that is not finite and >= 0 raise ValueError."""
        if temperatures is None:
            raise ValueError("thermal_conductivity_lbte needs temperatures")
        cutoff = float(pinv_cutoff)
        if not (math.isfinite(cutoff) and cutoff >= 0):
            raise ValueError(f"pinv_cutoff must be finite and non-negative, got {pinv_cutoff!r}")
        mesh, nu, e, n_imaginary, tets, temps = self._three_phonon_mesh(mesh, temperatures)
        iso, mfp = self._extra_scattering(mesh, nu, e, tets, mass_variances, boundary_mfp)
        n_mesh, nb = nu.shape
        dev, f64 = self.device, torch.float64
        t = torch.as_tensor(temps).to(dev)
        cols = torch.nonzero((nu >= THERMAL_CUTOFF_THZ).reshape(-1))[:, 0]
        m0 = len(cols)
        hot = [int(i) for i in np.nonzero(temps > 0)[0]]
        per_t = 8 * m0 * m0
        if hot and per_t > self.lbte_matrix_bytes:
            raise ValueError(f"thermal_conductivity_lbte needs {per_t} bytes for the collision matrix of one "
                             f"temperature ({m0} modes), more than lbte_matrix_bytes = {self.lbte_matrix_bytes}")
        per_group = max(1, self.lbte_matrix_bytes // max(per_t, 1))
        groups = [hot[i : i + per_group] for i in range(0, len(hot), per_group)] or [[]]
        avg = _degenerate_operators(nu)  # [N, 3n, 3n]
        pos = torch.full((n_mesh * nb,), -1, dtype=torch.long, device=dev)
        pos[cols] = torch.arange(m0, device=dev)
        gamma = torch.zeros(len(temps), n_mesh, nb, dtype=f64, device=dev)
        kappa = torch.zeros(len(temps), 3, 3, dtype=f64, device=dev)
        n_dropped = np.zeros(len(temps), dtype=np.int64)
        min_eig = np.full(len(temps), np.nan)
        res = x = s = total = None
        for group, target, g, rows in self._collision_passes(mesh, nu, e, tets, t, groups):
            if target == 0:
                s = torch.zeros(len(group), m0, m0, dtype=f64, device=dev)
            if g is not None:
                gamma[:, target] = g
            here = cols[(cols >= target * nb) & (cols < (target + 1) * nb)]
            for j in range(len(group)):  # per temperature, so that the grouping cannot change a bit
                rj = torch.einsum("ij,jcl->icl", avg[target], rows[j])
                rj = torch.einsum("icl,clk->ick", rj, avg).reshape(nb, -1)
                s[j, pos[here]] = rj[here - target * nb][:, cols]
            if target < n_mesh - 1:
                continue
            if res is None:  # the end of the first pass: every Gamma is known
                res, total = self._rta_conductivity(mesh, nu, gamma, t, temps, n_imaginary, iso, mfp)
                x = (torch.as_tensor(res["heat_capacity"]).to(dev).sqrt()[..., None]
                     * torch.as_tensor(res["group_velocities"]).to(dev)[None]).reshape(len(temps), -1, 3)[:, cols]
            for j, ti in enumerate(group):
                kappa[ti], n_dropped[ti], min_eig[ti] = self._lbte_solve(s[j], total[ti].reshape(-1)[cols], x[ti],
                                                                         cutoff)
            s = None
        vol = abs(float(np.linalg.det(self.cell.prim_lattice)))
        res["kappa_rta"] = res["kappa"]
        res["kappa"] = (kappa * (KAPPA_W_PER_MK / (n_mesh * vol))).cpu().numpy()
        res["n_dropped"], res["min_eigenvalue"] = n_dropped, min_eig
        return res

    @staticmethod
    def _lbte_solve(s, gamma, x, cutoff):
        """(sum over eta > cutoff of (U^T x)_k (x) (U^T x)_k / eta_k [3, 3], the count of eta <= cutoff, min eta) for
        Omega = diag(4 pi gamma) + (s + s^T) / 2 restricted to gamma > 0; s [M, M] averaged, gamma [M], x [M, 3]."""
        omega = (s + s.mT) * 0.5
        omega.diagonal().add_(4 * math.pi * gamma)
        keep = gamma > 0
        omega = omega[keep][:, keep]
        eta, u = torch.linalg.eigh(omega)
        y = u.mT @ x[keep]
        use = eta > cutoff
        k = (y[use] / eta[use, None]).mT @ y[use]
        return k, int((~use).sum()), float(eta.min()) if len(eta) else math.nan
