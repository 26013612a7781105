"""-m gpu: phonons on the device (CHGNet.phonons).

* ``chg_dynamical_matrices`` against its fp64 specification (oracle/phonons.py) at production sizes, with synthetic
  force constants: LiMnO2 4x4x4 on a 16^3 mesh, a 31-atom random cell 3x3x3 at random q, a non-diagonal supercell;
  bitwise reproducible;
* the device force constants against the fp64 oracle's and against the p2s rows of ``predict_hessian(supercell)``;
* Gamma against the live reference's Hessian (tests/golden/chgnet_0.3.0_hessian.npz); the commensurate q-points
  against the device supercell Hessian; ``thermal_properties`` against the host formula on spec frequencies."""
import os

import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import (THZ_PER_SQRT_EV_A2_AMU, gamma_mesh, make_supercell,
                                 thermal_properties_from_frequencies)
from oracle.phonons import PhononSpecKernels, oracle_compact_fcs

pytestmark = pytest.mark.gpu

# the fp32 device force constants against the fp64 oracle, as fractions of max|Phi| (TOL of test_hessian_gpu.py)
TOL = 2e-3


def _eigenvalues(nu):
    """eV/(A^2 amu) from THz, imaginary modes negative."""
    nu = np.asarray(nu)
    return np.sign(nu) * (nu / THZ_PER_SQRT_EV_A2_AMU) ** 2


@pytest.fixture(scope="module")
def model030():
    return phonon_cells.model030()


@pytest.fixture(scope="module")
def limno2_222(model030):
    return phonon_cells.limno2_222(model030)


@pytest.mark.parametrize("case", ["limno2_444_mesh16", "random31_333", "limno2_nondiagonal"])
def test_dynamical_matrices_kernel_matches_spec(case):
    from chgnet_b200._lib import CudaKernels

    rng = np.random.default_rng(17)
    if case == "limno2_444_mesh16":
        sc = make_supercell(*graphgen.limno2_structure(), [4, 4, 4])
        q = gamma_mesh((16, 16, 16))
    elif case == "random31_333":
        sc = make_supercell(*graphgen.random_structure(31, 9731), [3, 3, 3])
        q = rng.uniform(-1.0, 1.0, size=(300, 3))
    else:
        sc = make_supercell(*graphgen.limno2_structure(), [[1, 1, 0], [-1, 1, 0], [0, 0, 2]])
        q = rng.uniform(-0.5, 0.5, size=(1000, 3))
    mult = sc.multiplicities
    print(case, "atoms", len(sc.z), "q", len(q), "multiplicity histogram", np.bincount(mult.ravel()).tolist())
    if case.startswith("limno2"):  # pairs on the supercell boundary, with several minimum images, are reached
        assert mult.max() >= 4 and (mult > 1).sum() >= 100
    else:  # a random cell has no equidistant images: the production-size single-image path
        assert len(sc.z) == 837 and (mult == 1).all()
    n_prim, n = len(sc.p2s), len(sc.s2p)
    fc = rng.normal(size=(n_prim, n, 3, 3))
    dev = torch.device("cuda")
    args = [torch.as_tensor(x).to(dev) for x in (fc, sc.img_ptr, sc.img_vec, sc.s2p,
                                                   rng.uniform(0.1, 0.6, size=n_prim), q)]
    n3 = 3 * n_prim
    kern = CudaKernels(dev)
    got = torch.full((len(q), n3, n3), float("nan"), dtype=torch.complex128, device=dev)
    kern.dynamical_matrices(*args, got)
    again = torch.empty_like(got)
    kern.dynamical_matrices(*args, again)
    want = torch.empty_like(got)
    PhononSpecKernels().dynamical_matrices(*args, want)
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    print(case, f"max|D - spec| / max|D| = {err:.2e}")
    assert err <= 1e-10
    assert torch.equal(torch.view_as_real(got), torch.view_as_real(again))  # no atomics: bitwise reproducible
    assert torch.equal(got, got.conj().transpose(1, 2))  # written Hermitian


@pytest.mark.parametrize("cell", ["limno2_222", "random6_222"])
def test_device_force_constants_match_oracle(model030, weights030, limno2_222, cell):
    prim = graphgen.limno2_structure() if cell == "limno2_222" else graphgen.random_structure(6, 9741)
    ph = limno2_222 if cell == "limno2_222" else model030.phonons(prim, [2, 2, 2], batch_size=7)
    sc = ph.cell
    g = graphgen.make_crystal_graph(sc.z, sc.frac, sc.lattice)
    want = oracle_compact_fcs(weights030, g, sc.p2s)
    fc = ph.force_constants
    scale = np.abs(want).max()
    err = np.abs(fc - want).max() / scale
    h = model030.predict_hessian(g)
    n = len(sc.z)
    rows = h.reshape(n, 3, n, 3)[sc.p2s].transpose(0, 2, 1, 3)  # [n_prim, N, 3, 3]
    err_rows = np.abs(fc - rows).max() / scale
    print(cell, f"force constants vs oracle {err:.2e}, vs predict_hessian p2s rows {err_rows:.2e}, "
          f"asr_correction {ph.asr_correction:.2e} eV/A^2 (max|Phi| {scale:.2f})")
    assert fc.shape == (len(sc.p2s), n, 3, 3) and fc.dtype == np.float64
    assert err <= TOL and err_rows <= TOL


def test_gamma_matches_live_reference(limno2_222):
    with np.load(os.path.join(phonon_cells.GOLD, "chgnet_0.3.0_hessian.npz")) as f:
        h = f["limno2.hessian"]
    mw = 1.0 / np.sqrt(np.repeat(limno2_222.masses, 3))
    d = mw[:, None] * h * mw[None, :]
    want = np.linalg.eigvalsh(0.5 * (d + d.T))
    nu = limno2_222.frequencies([0.0, 0.0, 0.0])
    got = _eigenvalues(nu)
    err = np.abs(got - want).max() / np.abs(want).max()
    acoustic = np.sort(np.abs(nu))[:3]
    print(f"Gamma: eigenvalues vs reference {err:.2e} of the largest; acoustic |nu| {acoustic} THz; "
          f"lowest {nu[:2]} THz")
    assert err <= 2e-3
    assert acoustic.max() <= 1e-4
    assert (nu < -0.1).sum() == 1  # the unstable Gamma mode of this cell under 0.3.0 (DESIGN.md §12.1)


def test_commensurate_q_match_supercell_hessian(model030, limno2_222):
    sc = limno2_222.cell
    q = gamma_mesh((2, 2, 2))  # M = 2I: the 8 commensurate q-points
    nu, vec = limno2_222.frequencies(q, eigenvectors=True)
    assert nu.shape == (8, 24) and vec.shape == (8, 24, 24)
    assert np.abs(np.einsum("qij,qik->qjk", vec.conj(), vec) - np.eye(24)).max() < 1e-10
    got = np.sort(_eigenvalues(nu).ravel())
    h = model030.predict_hessian((sc.z, sc.frac, sc.lattice))
    mw = 1.0 / np.sqrt(np.repeat(limno2_222.masses[sc.s2p], 3))
    d = mw[:, None] * h * mw[None, :]
    want = np.linalg.eigvalsh(0.5 * (d + d.T))
    err = np.abs(got - want).max() / np.abs(want).max()
    print(f"commensurate q: eigenvalues vs supercell Hessian {err:.2e} of the largest")
    assert err <= 2e-3


def test_thermal_properties_match_host_formula(limno2_222):
    mesh, temps = (6, 6, 6), [0.0, 50.0, 300.0, 1000.0]
    got = limno2_222.thermal_properties(mesh, temps)
    spec = phonon_cells.spec_phonons(limno2_222.force_constants, limno2_222.cell)
    d = spec.dynamical_matrices(gamma_mesh(mesh)).numpy()
    lam = np.linalg.eigvalsh(d)
    want = thermal_properties_from_frequencies(np.sign(lam) * np.sqrt(np.abs(lam)) * THZ_PER_SQRT_EV_A2_AMU, temps)
    print("thermal", {k: v for k, v in got.items()})
    assert got["n_imaginary"] == want["n_imaginary"]
    for k in ("free_energy", "entropy", "heat_capacity", "zero_point_energy"):
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert np.abs(a - b).max() <= 1e-9 * max(np.abs(b).max(), 1e-12), k
