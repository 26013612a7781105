"""CPU (fp64): supercells and minimum images, compact force constants from Hessian-vector products, the dynamical-matrix
specification and the harmonic thermodynamics of chgnet_b200.phonons (CHGNet.phonons).

The force constants come from the kernel schedule with the torch specifications injected in fp64
(Engine + HessianSpecKernels) and from the oracle's double backward (oracle/phonons.py); D(q) from the specification of
``chg_dynamical_matrices`` (oracle/phonons.py)."""
import itertools

import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.dynamics import KB
from chgnet_b200.engine import Engine
from chgnet_b200.phonons import (H_EV_PER_THZ, THZ_PER_SQRT_EV_A2_AMU, compact_force_constants, make_supercell,
                                 thermal_properties_from_frequencies)
from chgnet_b200.weights import pack_weights
from oracle.hessian import HessianSpecKernels, oracle_hessian
from oracle.phonons import oracle_compact_fcs

SKEWED = [[1, 3, 0], [0, 1, 0], [0, 0, 2]]
NONDIAG = [[1, 1, 0], [-1, 1, 0], [0, 0, 1]]


def spec_hvp(weights):
    sd = {k: torch.as_tensor(np.asarray(v)).double() for k, v in weights.items()}
    eng = Engine(pack_weights(sd, None, device="cpu", dtype=torch.float64), HessianSpecKernels())

    def hvp(graph, v):
        k, n = v.shape[0], v.shape[1]
        b = build_batch([graph] * k, "cpu")
        b.frac, b.lattice, b.image = b.frac.double(), b.lattice.double(), b.image.double()
        return eng.hessian_vector_products(b, torch.as_tensor(v).reshape(k * n, 3)).view(k, n, 3).numpy()

    return hvp


def commensurate_qpoints(m) -> np.ndarray:
    """The det M reduced q-points with M q integral (e^{2 pi i q.T} = 1 for every supercell translation T)."""
    m = np.asarray(m, dtype=np.float64)
    det = int(round(np.linalg.det(m)))
    q = np.array([np.linalg.solve(m, k) for k in itertools.product(range(det), repeat=3)])
    q = np.round(q - np.floor(q + 1e-9), 9) % 1.0
    q = np.unique(q, axis=0)
    assert len(q) == det
    return q


def brute_force_images(sc, reach=4):
    """Minimum images of every (k, j) pair over +-reach supercell translations, in primitive fractional coordinates."""
    t = np.array(list(itertools.product(range(-reach, reach + 1), repeat=3)), dtype=np.float64)
    out = {}
    for k, k0 in enumerate(sc.p2s):
        for j in range(len(sc.s2p)):
            v = (sc.frac[j] - sc.frac[k0])[None, :] + t  # supercell fractional
            length = np.linalg.norm(v @ sc.lattice, axis=1)
            keep = v[length <= length.min() + 1e-5] @ sc.matrix
            out[k, j] = keep[np.lexsort(keep.T[::-1])]
    return out


@pytest.mark.parametrize("cell", ["limno2", "random5"])
@pytest.mark.parametrize("m", [[2, 2, 2], [2, 1, 3], NONDIAG, SKEWED])
def test_supercell_atoms_maps_and_images(cell, m):
    z, frac, lat = graphgen.limno2_structure() if cell == "limno2" else graphgen.random_structure(5, 77)
    sc = make_supercell(z, frac, lat, m)
    det = int(round(np.linalg.det(np.diag(m) if np.ndim(m) == 1 else np.asarray(m))))
    n_prim, n_cells = len(z), det
    assert len(sc.z) == n_prim * det and sc.points.shape == (n_cells, 3) and not sc.points[0].any()
    assert np.allclose(sc.lattice, sc.matrix @ lat)
    # unique modulo the supercell lattice
    diff = sc.frac[:, None, :] - sc.frac[None, :, :]
    is_same = np.all(np.abs(diff - np.round(diff)) < 1e-8, axis=2)
    assert (is_same.sum(axis=1) == 1).all()
    # r_j = r_k + R_l (modulo the supercell lattice) for j = k n_cells + l
    minv = np.linalg.inv(sc.matrix.astype(np.float64))
    for j in range(len(sc.z)):
        k, l = divmod(j, n_cells)
        x = (frac[k] + sc.points[l]) @ minv - sc.frac[j]
        assert np.abs(x - np.round(x)).max() < 1e-10
        assert sc.s2p[j] == k and sc.z[j] == z[k]
    assert (sc.s2p[sc.p2s] == np.arange(n_prim)).all() and (sc.p2s == np.arange(n_prim) * n_cells).all()
    # the minimum-image table equals a brute-force search over +-4 supercell translations
    want = brute_force_images(sc)
    for (k, j), w in want.items():
        got = sc.img_vec[sc.img_ptr[k * len(sc.z) + j] : sc.img_ptr[k * len(sc.z) + j + 1]]
        got = got[np.lexsort(got.T[::-1])]
        assert got.shape == w.shape and np.abs(got - w).max() < 1e-9, (k, j, got, w)


def test_multiplicities_on_limno2_222():
    sc = make_supercell(*graphgen.limno2_structure(), [2, 2, 2])
    mult = sc.multiplicities
    assert mult.min() == 1 and mult.max() == 8 and (mult > 1).sum() > 0


@pytest.mark.parametrize("m", [[[1, 0, 0], [0, 1, 0], [0, 0, -1]], [2, 0, 1], [1.5, 1, 1], np.eye(2)])
def test_bad_supercell_matrix(m):
    with pytest.raises(ValueError):
        make_supercell(*graphgen.limno2_structure(), m)


@pytest.fixture(scope="module")
def limno2_211(weights030):
    sc, g, fc = phonon_cells.limno2_211(weights030)
    return sc, g, oracle_hessian(weights030, g), fc


def test_translation_identity_of_oracle_supercell_hessian(limno2_211):
    sc, _, h, _ = limno2_211
    n, n_cells = len(sc.z), len(sc.points)
    scale = np.abs(h).max()
    minv = np.linalg.inv(sc.matrix.astype(np.float64))
    hb = h.reshape(n, 3, n, 3)
    for j in range(n):
        k, l = divmod(j, n_cells)
        # translation by -R_l: atom i goes to the atom at r_i - R_l
        shifted = sc.frac - sc.points[l] @ minv
        d = shifted[:, None, :] - sc.frac[None, :, :]
        perm = np.argmax(np.all(np.abs(d - np.round(d)) < 1e-8, axis=2), axis=1)
        assert sorted(perm) == list(range(n))
        row0 = hb[sc.p2s[k]]  # [3, n, 3]
        assert np.abs(hb[j] - row0[:, perm]).max() <= 1e-10 * scale


def test_spec_engine_force_constants_match_oracle(weights030, limno2_211):
    hvp = spec_hvp(weights030)
    sc, g, _, want = limno2_211
    got = compact_force_constants(lambda v: hvp(g, v), sc)
    assert got.shape == (8, 16, 3, 3)
    assert np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
    sc1 = make_supercell(*phonon_cells.CU, [2, 2, 2])
    g1 = graphgen.make_crystal_graph(sc1.z, sc1.frac, sc1.lattice)
    want1 = oracle_compact_fcs(weights030, g1, sc1.p2s)
    got1 = compact_force_constants(lambda v: hvp(g1, v), sc1)
    assert got1.shape == (1, 8, 3, 3) and np.abs(want1).max() > 1e-2
    assert np.abs(got1 - want1).max() <= 1e-6 * np.abs(want1).max()


def _spec_dyn(fc, sc, q):
    ph = phonon_cells.spec_phonons(fc, sc)
    ph._fc = torch.as_tensor(fc)  # the identities hold for the force constants as computed (no ASR correction)
    return ph.dynamical_matrices(q).numpy(), ph.masses


@pytest.mark.parametrize("m", [[2, 1, 1], NONDIAG])
def test_exact_identities_of_the_dynamical_matrix(weights030, limno2_211, m):
    z, frac, lat = graphgen.limno2_structure()
    if m == [2, 1, 1]:
        sc, _, h_super, fc = limno2_211
    else:
        sc = make_supercell(z, frac, lat, m)
        g = graphgen.make_crystal_graph(sc.z, sc.frac, sc.lattice)
        h_super, fc = oracle_hessian(weights030, g), oracle_compact_fcs(weights030, g, sc.p2s)
    # D(Gamma) = M^-1/2 H_prim M^-1/2
    d, masses = _spec_dyn(fc, sc, np.zeros((1, 3)))
    mw = 1.0 / np.sqrt(np.repeat(masses, 3))
    want = mw[:, None] * oracle_hessian(weights030, graphgen.make_crystal_graph(z, frac, lat)) * mw[None, :]
    assert np.abs(d[0] - want).max() <= 1e-9 * np.abs(want).max()
    # over the commensurate q-points, the eigenvalues of D(q) are those of the mass-weighted supercell Hessian
    q = commensurate_qpoints(sc.matrix)
    d, _ = _spec_dyn(fc, sc, q)
    got = np.sort(np.linalg.eigvalsh(d).ravel())
    ms = 1.0 / np.sqrt(np.repeat(masses[sc.s2p], 3))
    hs = ms[:, None] * h_super * ms[None, :]
    want = np.sort(np.linalg.eigvalsh(0.5 * (hs + hs.T)))
    assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()


def test_frequencies_path_with_spec_kernels(limno2_211):
    sc, _, _, fc = limno2_211
    ph = phonon_cells.spec_phonons(fc, sc)
    assert ph.supercell[0].shape == (16,) and ph.asr_correction < 1e-9 * np.abs(fc).max()
    rng = np.random.default_rng(3)
    q = np.vstack([np.zeros(3), rng.uniform(-0.5, 0.5, size=(6, 3))])
    nu, vec = ph.frequencies(q, eigenvectors=True)
    assert nu.shape == (7, 24) and vec.shape == (7, 24, 24) and (np.diff(nu, axis=1) >= 0).all()
    assert np.abs(nu[0, 1:4]).max() < 1e-4 and nu[0, 0] < -0.1  # three acoustic modes and the unstable Gamma mode
    d = ph.dynamical_matrices(q).numpy()
    lam = np.sign(nu) * (nu / THZ_PER_SQRT_EV_A2_AMU) ** 2
    assert np.abs(d @ vec - vec * lam[:, None, :]).max() <= 1e-10 * np.abs(d).max()
    assert np.abs(np.einsum("qij,qik->qjk", vec.conj(), vec) - np.eye(24)).max() < 1e-12
    ph.chunk_bytes = 3 * 24 * 24 * 16  # three q-points per chunk
    def lam_of(f):
        return np.sign(f) * f**2

    assert np.abs(lam_of(ph.frequencies(q)) - lam_of(nu)).max() <= 1e-12 * np.abs(lam_of(nu)).max()
    assert np.abs(lam_of(ph.frequencies(q[3])) - lam_of(nu[3])).max() <= 1e-12 * np.abs(lam_of(nu)).max()


def test_einstein_solid():
    nu, n_modes = 5.0, 12
    temps = np.array([0.0, 10.0, 300.0, 2000.0])
    out = thermal_properties_from_frequencies(np.full((4, n_modes), nu), temps)
    e = H_EV_PER_THZ * nu
    x = e / (KB * temps[1:])
    f = n_modes * (e / 2 + KB * temps[1:] * np.log(1 - np.exp(-x)))
    s = n_modes * KB * (x / (np.exp(x) - 1) - np.log(1 - np.exp(-x)))
    c = n_modes * KB * x**2 * np.exp(x) / (np.exp(x) - 1) ** 2
    assert abs(out["zero_point_energy"] - n_modes * e / 2) <= 1e-12 * n_modes * e
    assert out["free_energy"][0] == out["zero_point_energy"] and out["entropy"][0] == 0 and out["heat_capacity"][0] == 0
    for got, want in ((out["free_energy"][1:], f), (out["entropy"][1:], s), (out["heat_capacity"][1:], c)):
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    assert out["n_imaginary"] == 0


def test_thermal_high_temperature_limit_and_cutoff():
    rng = np.random.default_rng(5)
    n_prim = 4
    nu = np.sort(rng.uniform(1.0, 15.0, size=(50, 3 * n_prim)), axis=1)
    nu[0, :3] = [-2e-3, 0.0, 5e-4]  # one imaginary mode, two left out
    out = thermal_properties_from_frequencies(nu, [1e6])  # x = h nu / kT < 1e-3
    kept = (nu >= 1e-3).sum() / 50
    assert out["n_imaginary"] == 1
    assert abs(out["heat_capacity"][0] - kept * KB) <= 1e-6 * kept * KB
    assert abs(kept - 3 * n_prim) < 0.1
