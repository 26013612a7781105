"""CPU (fp64): thermal displacement matrices of chgnet_b200.phonons (Phonons.thermal_displacement_matrices), with the
specification of ``chg_thermal_displacements`` (oracle/phonons.py).

* the specification against a plain triple loop, and the Einstein identity;
* simple cubic and orthorhombic crystals of nearest-neighbour central springs (three independent 1D chains): the exact
  finite-mesh sums, on 3x3x3 and 2x2x2 supercells;
* the Cartesian -> CIF conversion on a triclinic lattice;
* the commensurate identity: on the mesh M, U is the diagonal block of a matrix function of the mass-weighted
  supercell Hessian (LiMnO2 2x1x1 with the oracle's force constants, and the spring crystal);
* limits (convergence with the mesh on a one-atom fcc spring crystal, the classical limit, monotonicity in T) and
  bookkeeping (the Gamma acoustic exclusion under force-constant noise, the imaginary part of the complex sum, chunking,
  ``n_imaginary``, bad temperatures)."""
import numpy as np
import pytest
import torch

from chgnet_b200.phonons import (DISPLACEMENT_A2_AMU_THZ, H_OVER_KB_K_PER_THZ, THERMAL_CUTOFF_THZ,
                                 THZ_PER_SQRT_EV_A2_AMU, acoustic_sum_rule, cif_displacement_matrices, gamma_mesh,
                                 make_supercell)
from oracle.phonons import PhononSpecKernels
from oracle.thermal_displacements import VOIGT
from phonon_cells import CU, K, limno2_211_spec, spec_phonons, springs

C = DISPLACEMENT_A2_AMU_THZ
TEMPS = np.array([0.0, 10.0, 300.0, 1500.0])


def _unitary(rng, n, size):
    z = rng.normal(size=(size, n, n)) + 1j * rng.normal(size=(size, n, n))
    return np.linalg.qr(z)[0]  # [size, n, n], columns orthonormal


def _coth_over_nu(nu, t):
    """coth(h nu / 2 k T) / nu, computed independently of the specification (1 / nu at T = 0)."""
    return (1.0 / np.tanh(H_OVER_KB_K_PER_THZ * nu / (2 * t)) if t > 0 else 1.0) / nu


def _spec_sums(freqs, vecs, temps):
    acc = torch.zeros(len(temps), freqs.shape[1] // 3, 6, dtype=torch.float64)
    PhononSpecKernels().thermal_displacements(torch.as_tensor(freqs), torch.as_tensor(vecs), torch.as_tensor(temps),
                                              THERMAL_CUTOFF_THZ, acc)
    return acc.numpy()


def test_spec_matches_triple_loop():
    rng = np.random.default_rng(41)
    n_q, n_prim = 5, 2
    n3 = 3 * n_prim
    u = _unitary(rng, n3, n_q)  # column m: mode m
    nu = rng.uniform(-3.0, 12.0, size=(n_q, n3))
    nu[0, :3] = [0.0, 5e-4, -2e-3]  # below the cutoff, and imaginary
    nu[1, 0] = THERMAL_CUTOFF_THZ  # on the cutoff: kept
    got = _spec_sums(nu, np.ascontiguousarray(u.transpose(0, 2, 1)), TEMPS)
    want = np.zeros((len(TEMPS), n_prim, 6))
    for q in range(n_q):
        for m in range(n3):
            if nu[q, m] < THERMAL_CUTOFF_THZ:
                continue
            for t, temp in enumerate(TEMPS):
                w = (1.0 + (2.0 / np.expm1(H_OVER_KB_K_PER_THZ * nu[q, m] / temp) if temp > 0 else 0.0)) / nu[q, m]
                for k in range(n_prim):
                    e = u[q, 3 * k : 3 * k + 3, m]
                    outer = np.real(np.outer(e, e.conj()))
                    want[t, k] += w * outer[VOIGT[0], VOIGT[1]]
    err = np.abs(got - want).max() / np.abs(want).max()
    print(f"specification vs triple loop: {err:.1e}")
    assert err <= 1e-14


def test_einstein_identity():
    rng = np.random.default_rng(43)
    n_q, n_prim, nu0 = 7, 3, 4.2
    u = _unitary(rng, 3 * n_prim, n_q)
    got = _spec_sums(np.full((n_q, 3 * n_prim), nu0), np.ascontiguousarray(u.transpose(0, 2, 1)), TEMPS) / n_q
    for t, temp in enumerate(TEMPS):
        want = _coth_over_nu(nu0, temp) * np.array([1.0, 1, 1, 0, 0, 0])
        assert np.abs(got[t] - want).max() <= 1e-13 * np.abs(want).max()


def _chain_sum(nu_max, n, t):
    """(1/n) sum_{j=1}^{n-1} coth(h nu_j / 2 k T) / nu_j, nu_j = nu_max sin(pi j / n)."""
    return _coth_over_nu(nu_max * np.sin(np.pi * np.arange(1, n) / n), t).sum() / n


@pytest.mark.parametrize("crystal", ["cubic_333", "cubic_222", "orthorhombic_333"])
@pytest.mark.parametrize("n", [4, 7, 8])
def test_spring_crystal_exact_mesh_sums(crystal, n):
    if crystal == "orthorhombic_333":
        ph, nu_max = springs([3, 3, 3], ks=(3.0, 1.7, 4.4), a=(2.7, 3.1, 2.4))
    else:
        ph, nu_max = springs([3, 3, 3] if crystal == "cubic_333" else [2, 2, 2])
    out = ph.thermal_displacement_matrices((n, n, n), TEMPS)
    u = out["cartesian"]
    assert u.shape == (4, 1, 3, 3) and out["cif"].shape == (4, 1, 3, 3) and out["n_imaginary"] == 0
    assert (out["temperatures"] == TEMPS).all()
    for t, temp in enumerate(TEMPS):
        want = np.diag([C / ph.masses[0] * _chain_sum(nu_max[c], n, temp) for c in range(3)])
        assert np.abs(u[t, 0] - want).max() <= 1e-12 * np.abs(want).max()
    assert np.abs(out["cif"] - u).max() <= 1e-15 * np.abs(u).max()


def test_cif_conversion():
    rng = np.random.default_rng(47)
    lat = np.array([[3.1, 0.2, -0.3], [0.7, 4.0, 0.4], [-0.5, 1.1, 5.2]])  # triclinic, rows are lattice vectors
    recip = np.linalg.inv(lat).T
    unit = recip / np.linalg.norm(recip, axis=1)[:, None]
    cosines = unit @ unit.T
    assert np.abs(cosines - np.eye(3)).max() > 0.05
    u = 0.013
    got = cif_displacement_matrices(u * np.eye(3), lat)
    err = np.abs(got - u * cosines).max()
    print(f"isotropic u I -> u cos(a*_i, a*_j): {err:.1e}")
    assert err <= 1e-16
    # a random symmetric U round-trips through U = A N U_cif N A^T
    x = rng.normal(size=(5, 3, 3))
    uc = 0.01 * (x + x.transpose(0, 2, 1))
    cif = cif_displacement_matrices(uc, lat)
    a_n = lat.T * np.linalg.norm(recip, axis=1)[None, :]
    assert np.abs(a_n @ cif @ a_n.T - uc).max() <= 1e-15 * np.abs(uc).max() * 10
    assert np.abs(cif - cif.transpose(0, 2, 1)).max() <= 1e-17
    # U_eq = (1/3) sum_ij U^cif_ij a*_i a*_j (a_i . a_j) = trace(U_cart) / 3
    metric = lat @ lat.T
    norms = np.linalg.norm(recip, axis=1)
    u_eq = np.einsum("qij,i,j,ij->q", cif, norms, norms, metric) / 3
    assert np.abs(u_eq - np.trace(uc, axis1=1, axis2=2) / 3).max() <= 1e-15


def _supercell_displacements(ph, temps):
    """[T, N, 3, 3] diagonal blocks of (C / m) M^-1/2 g(H) M^-1/2 over the supercell: H the mass-weighted Hessian
    assembled by lattice translation from the acoustic-sum-rule-corrected compact force constants, its three
    translation modes projected out, g = coth(h nu / 2 k T) / nu over the modes with nu >= the cutoff."""
    sc = ph.cell
    n, n_cells = len(sc.z), len(sc.points)
    fc, _ = acoustic_sum_rule(ph.force_constants, sc.p2s)
    minv = np.linalg.inv(sc.matrix.astype(np.float64))
    h = np.zeros((n, 3, n, 3))
    for j in range(n):
        k, l = divmod(j, n_cells)
        shifted = sc.frac - sc.points[l] @ minv  # the atom at r_i - R_l, for every i
        d = shifted[:, None, :] - sc.frac[None, :, :]
        perm = np.argmax(np.all(np.abs(d - np.round(d)) < 1e-8, axis=2), axis=1)
        h[j] = fc[k][perm].transpose(1, 0, 2)  # Phi(k l, i) = Phi(k 0, atom of r_i - R_l)
    h = h.reshape(3 * n, 3 * n)
    m = np.repeat(ph.masses[sc.s2p], 3)
    hm = h / np.sqrt(m)[:, None] / np.sqrt(m)[None, :]
    hm = 0.5 * (hm + hm.T)
    trans = np.zeros((3 * n, 3))
    for c in range(3):
        trans[c::3, c] = np.sqrt(ph.masses[sc.s2p])
    trans /= np.linalg.norm(trans, axis=0)
    basis = np.linalg.svd(np.eye(3 * n) - trans @ trans.T)[0][:, : 3 * n - 3]  # the complement of the translations
    lam, w = np.linalg.eigh(basis.T @ hm @ basis)
    vec = basis @ w
    nu = np.sign(lam) * np.sqrt(np.abs(lam)) * THZ_PER_SQRT_EV_A2_AMU
    keep = nu >= THERMAL_CUTOFF_THZ
    out = np.zeros((len(temps), n, 3, 3))
    for t, temp in enumerate(temps):
        g = np.zeros_like(nu)
        g[keep] = _coth_over_nu(nu[keep], temp)
        blocks = np.einsum("s,is,js->ij", g, vec, vec).reshape(n, 3, n, 3)
        out[t] = blocks[np.arange(n), :, np.arange(n), :] * (C / m[::3])[:, None, None]
    return out, nu


@pytest.fixture(scope="module")
def limno2_211(weights030):
    return limno2_211_spec(weights030)


@pytest.mark.parametrize("crystal", ["limno2_211", "springs_333"])
def test_commensurate_identity(crystal, request):
    ph = request.getfixturevalue("limno2_211") if crystal == "limno2_211" else springs([3, 3, 3])[0]
    mesh = np.diag(ph.cell.matrix)
    temps = np.array([0.0, 300.0, 1000.0])
    out = ph.thermal_displacement_matrices(mesh, temps)
    want, nu_super = _supercell_displacements(ph, temps)
    n_cells = len(ph.cell.points)
    scale = np.abs(want).max()
    for l in range(n_cells):  # every copy of atom k carries the same block
        err = np.abs(out["cartesian"] - want[:, l::n_cells]).max() / scale
        assert err <= 1e-10, (l, err)
    print(f"{crystal}: mesh {mesh.tolist()} vs supercell matrix function, max/scale over copies "
          f"{max(np.abs(out['cartesian'] - want[:, l::n_cells]).max() for l in range(n_cells)) / scale:.1e}; "
          f"n_imaginary {out['n_imaginary']}, supercell modes below -cutoff {(nu_super < -THERMAL_CUTOFF_THZ).sum()}")
    if crystal == "limno2_211":  # the imaginary mode is left out on both sides
        assert out["n_imaginary"] >= 1 and (nu_super < -THERMAL_CUTOFF_THZ).sum() == out["n_imaginary"]


def _fcc_springs(m, doubled=False, noise=0.0, seed=0):
    """One atom per fcc primitive cell (a = 3.61 A), nearest-neighbour central springs K; with ``doubled`` the primitive
    cell is two fcc cells (lattice rows 2 a1, a2, a3), and ``noise`` adds Gaussian noise that is not symmetric."""
    lat1 = CU[2]
    lat, frac = (lat1 * [[2], [1], [1]], [[0.0, 0, 0], [0.5, 0, 0]]) if doubled else (lat1, [[0.0, 0, 0]])
    sc = make_supercell([29] * len(frac), np.asarray(frac), lat, m)
    n = len(sc.z)
    fc = np.zeros((len(frac), n, 3, 3))
    nbrs = [np.array(v) for v in ([1, 0, 0], [0, 1, 0], [0, 0, 1], [1, -1, 0], [1, 0, -1], [0, 1, -1])]
    inv = np.linalg.inv(sc.lattice)
    for k, k0 in enumerate(sc.p2s):
        for v in nbrs + [-v for v in nbrs]:
            r = v @ lat1
            x = ((sc.frac[k0] @ sc.lattice + r) @ inv) % 1.0
            j = int(np.argmin(np.abs((sc.frac - x + 0.5) % 1.0 - 0.5).sum(1)))
            phi = K * np.outer(r, r) / (r @ r)
            fc[k, j] -= phi
            fc[k, k0] += phi
    if noise:
        fc += noise * np.random.default_rng(seed).normal(size=fc.shape)
    return spec_phonons(fc, sc)


def test_limits():
    # convergence with the mesh on a 3D model with a finite limit
    ph = _fcc_springs([4, 4, 4])
    assert (ph.cell.multiplicities[0][np.abs(ph.force_constants[0]).sum(axis=(1, 2)) > 0] == 1).all()
    u = [ph.thermal_displacement_matrices((n, n, n), [300.0])["cartesian"][0, 0] for n in (8, 16, 32)]
    diffs = [np.abs(u[1] - u[0]).max(), np.abs(u[2] - u[1]).max()]
    print(f"fcc springs at 300 K: U_xx on 8^3, 16^3, 32^3 = {[float(x[0, 0]) for x in u]} A^2, "
          f"successive differences {diffs}")
    # cubic: isotropic on every mesh
    for x in u:
        assert np.abs(x - x[0, 0] * np.eye(3)).max() <= 1e-12 * x[0, 0]
    # calibrated on this model (differences 2.0e-4 and 9.9e-5 A^2, ratio 0.51): the mesh samples the region around
    # Gamma, where the weight grows as 1/nu^2, with an error that falls as 1/n
    assert diffs[1] < 0.6 * diffs[0] and diffs[1] <= 1.2e-4

    # classical limit: U / T -> (k / N_q m) sum e e^H / omega^2, relative gap ~ (h nu / k T)^2 / 12
    ph, nu_max = springs([3, 3, 3], ks=(3.0, 1.7, 4.4), a=(2.7, 3.1, 2.4))
    mesh = (5, 5, 5)
    temps = np.array([2000.0, 4000.0, 8000.0])
    u = ph.thermal_displacement_matrices(mesh, temps)["cartesian"][:, 0]
    classical = np.diag([C / ph.masses[0] / 5 * (2 / (H_OVER_KB_K_PER_THZ
                                                      * (nu_max[c] * np.sin(np.pi * np.arange(1, 5) / 5)) ** 2)).sum()
                         for c in range(3)])  # per K
    gaps = [np.abs(u[t] / temps[t] - classical).max() / np.abs(classical).max() for t in range(3)]
    x_max = [H_OVER_KB_K_PER_THZ * nu_max.max() / t for t in temps]
    print("classical limit: relative gaps", gaps, "bounds (h nu_max / k T)^2 / 12", [x * x / 12 for x in x_max])
    for g, x in zip(gaps, x_max):
        assert 0 < g <= x * x / 12
    assert 0.2 <= gaps[1] / gaps[0] <= 0.3 and 0.2 <= gaps[2] / gaps[1] <= 0.3

    # non-decreasing in T: U(T2) - U(T1) is positive semi-definite
    temps = np.linspace(0.0, 1500.0, 31)
    u = ph.thermal_displacement_matrices(mesh, temps)["cartesian"][:, 0]
    ev = np.linalg.eigvalsh(np.diff(u, axis=0))
    assert ev.min() >= -1e-15 * np.abs(u).max()
    assert (np.diff(np.trace(u, axis1=1, axis2=2)) > 0).all()


def test_gamma_acoustic_exclusion_under_noise():
    # two atoms per primitive cell (the fcc spring crystal, doubled): with force constants that are not symmetric,
    # the acoustic-sum-rule correction leaves a small non-zero acoustic block in D(Gamma)
    clean = _fcc_springs([2, 3, 3], doubled=True)
    noise = 3e-3 * K  # the acoustic block of D(Gamma) grows with the part of the noise that is not symmetric
    noisy = _fcc_springs([2, 3, 3], doubled=True, noise=noise, seed=0)
    nu_gamma = np.sort(np.abs(noisy.frequencies([0.0, 0.0, 0.0])))
    print("Gamma |nu| with noise (THz):", nu_gamma)
    nu_gamma = nu_gamma[:3]
    assert nu_gamma.min() > 10 * THERMAL_CUTOFF_THZ  # above the cutoff: only the Gamma rule leaves them out
    assert np.sort(np.abs(clean.frequencies([0.0, 0.0, 0.0])))[2] < THERMAL_CUTOFF_THZ
    mesh, temps = (4, 4, 4), np.array([0.0, 300.0, 1000.0])
    u0 = clean.thermal_displacement_matrices(mesh, temps)["cartesian"]
    u1 = noisy.thermal_displacement_matrices(mesh, temps)["cartesian"]
    change = np.abs(u1 - u0).max() / np.abs(u0).max()
    # what the three Gamma modes would add if they were kept: ~ 2 k T / (h nu^2) each
    kept = C / noisy.masses[0] / 64 * _coth_over_nu(nu_gamma, 1000.0).sum()
    print(f"Gamma acoustic |nu| under noise {nu_gamma} THz; relative change of U {change:.1e}; "
          f"the three modes would add {kept:.2e} A^2 at 1000 K against max U {np.abs(u0).max():.2e}")
    assert change <= 10 * noise / K
    assert kept >= 100 * np.abs(u0).max()


def test_imaginary_part_of_the_full_sum(limno2_211):
    ph = limno2_211
    mesh = (4, 3, 2)
    q = gamma_mesh(mesh)
    nu, vec = ph.frequencies(q, eigenvectors=True)
    w = np.where(nu >= THERMAL_CUTOFF_THZ, 1.0 / np.where(nu >= THERMAL_CUTOFF_THZ, nu, 1.0), 0.0)
    e = vec.reshape(len(q), 8, 3, 24)  # [q, atom, alpha, mode]
    full = np.einsum("qm,qkam,qkbm->kab", w, e, e.conj())
    ratio = np.abs(full.imag).max() / np.abs(full.real).max()
    print(f"LiMnO2 2x1x1, mesh {mesh}: max|Im| / max|Re| of the complex sum = {ratio:.1e}")
    assert ratio <= 1e-13


def test_chunking_n_imaginary_and_bad_temperatures(limno2_211):
    ph = limno2_211
    mesh, temps = (3, 4, 2), np.array([0.0, 150.0, 300.0, 1200.0])
    whole = ph.thermal_displacement_matrices(mesh, temps)
    chunked = spec_phonons(ph.force_constants, ph.cell)
    chunked.eigh_batch = 5  # Gamma in the first chunk, a short last chunk
    small = chunked.thermal_displacement_matrices(mesh, temps)
    assert np.abs(small["cartesian"] - whole["cartesian"]).max() <= 1e-13 * np.abs(whole["cartesian"]).max()
    chunked.eigh_batch, chunked.chunk_bytes = 4096, 3 * 24 * 24 * 16
    small = chunked.thermal_displacement_matrices(mesh, temps)
    assert np.abs(small["cartesian"] - whole["cartesian"]).max() <= 1e-13 * np.abs(whole["cartesian"]).max()
    nu = ph.frequencies(gamma_mesh(mesh))
    assert whole["n_imaginary"] == int((nu < -THERMAL_CUTOFF_THZ).sum()) >= 1
    assert whole["n_imaginary"] == ph.thermal_properties(mesh, [300.0])["n_imaginary"]
    u = whole["cartesian"]
    assert np.abs(u - u.transpose(0, 1, 3, 2)).max() == 0
    assert (np.linalg.eigvalsh(u) > 0).all()
    for bad in ([-1.0], [300.0, np.nan], [np.inf]):
        with pytest.raises(ValueError):
            ph.thermal_displacement_matrices(mesh, bad)
    with pytest.raises(ValueError):
        ph.thermal_displacement_matrices((0, 2, 2), [300.0])
