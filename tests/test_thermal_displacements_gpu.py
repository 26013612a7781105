"""-m gpu: thermal displacement matrices on the device (Phonons.thermal_displacement_matrices).

* ``chg_thermal_displacements`` against its fp64 specification (oracle/phonons.py) at production sizes:
  4 096 q x 24 modes x 31 temperatures, the 31-atom cell's 93 modes, one temperature, one atom, 300 temperatures (two
  temperature tiles); bitwise reproducible, exact doubling on a second accumulation, and the Einstein identity;
* the device force constants of LiMnO2 2x2x2 on a 20^3 mesh (two eigh chunks): the device path against the
  specification path on the same force constants;
* fcc Cu 4x4x4 (0.3.0 weights): U at 300 K on 8^3, 16^3 and 24^3 meshes, cubic isotropy and the CIF form."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200.phonons import H_OVER_KB_K_PER_THZ, THERMAL_CUTOFF_THZ
from oracle.phonons import PhononSpecKernels
from phonon_cells import CU

pytestmark = pytest.mark.gpu

TEMPS = np.linspace(0.0, 1500.0, 31)


def _random_modes(n_q, n_prim, seed, equal=None):
    """Random unitary eigenvectors [n_q, mode, 3n] (mode-major) and frequencies [n_q, 3n] on the device: negative
    values, values below the cutoff, and the cutoff itself included; ``equal`` makes every frequency that value."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n3 = 3 * n_prim
    z = torch.complex(torch.randn(n_q, n3, n3, generator=g, device="cuda", dtype=torch.float64),
                      torch.randn(n_q, n3, n3, generator=g, device="cuda", dtype=torch.float64))
    e = torch.linalg.qr(z)[0].mT.contiguous()  # row m: mode m
    if equal is not None:
        return torch.full((n_q, n3), equal, dtype=torch.float64, device="cuda"), e
    nu = torch.rand(n_q, n3, generator=g, device="cuda", dtype=torch.float64) * 23.0 - 3.0
    nu[:, 0] = 0.0
    nu[::3, 1] = 5e-4
    nu[1::3, 1] = THERMAL_CUTOFF_THZ
    nu[2::3, 1] = -1e-2
    return nu, e


@pytest.mark.parametrize("case", ["8atoms_4096q_31T", "31atoms_1024q_31T", "8atoms_4096q_1T", "1atom_5000q_31T",
                                  "2atoms_2000q_300T"])
def test_kernel_matches_spec(case):
    from chgnet_b200._lib import CudaKernels

    n_prim, n_q, n_t = {"8atoms_4096q_31T": (8, 4096, 31), "31atoms_1024q_31T": (31, 1024, 31),
                        "8atoms_4096q_1T": (8, 4096, 1), "1atom_5000q_31T": (1, 5000, 31),
                        "2atoms_2000q_300T": (2, 2000, 300)}[case]
    nu, e = _random_modes(n_q, n_prim, seed=n_prim * 1000 + n_t)
    temps = TEMPS if n_t == 31 else (np.array([300.0]) if n_t == 1 else np.linspace(0.0, 3000.0, n_t))
    t = torch.as_tensor(temps).cuda()
    kern = CudaKernels("cuda")

    def run(k, acc=None):
        acc = torch.zeros(n_t, n_prim, 6, dtype=torch.float64, device="cuda") if acc is None else acc
        k.thermal_displacements(nu, e, t, THERMAL_CUTOFF_THZ, acc)
        return acc

    got, want = run(kern), run(PhononSpecKernels())
    again = run(kern)
    twice = run(kern, got.clone())
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    print(f"{case}: max|kernel - spec| / max = {err:.2e} (max {scale:.3e})")
    assert err <= 1e-12
    assert torch.equal(got, again)
    assert torch.equal(twice, 2 * got)


def test_kernel_einstein_identity():
    from chgnet_b200._lib import CudaKernels

    n_q, n_prim, nu0 = 4096, 8, 4.2
    nu, e = _random_modes(n_q, n_prim, seed=5, equal=nu0)
    acc = torch.zeros(len(TEMPS), n_prim, 6, dtype=torch.float64, device="cuda")
    CudaKernels("cuda").thermal_displacements(nu, e, torch.as_tensor(TEMPS).cuda(), THERMAL_CUTOFF_THZ, acc)
    got = acc.cpu().numpy() / n_q
    coth = np.array([1.0] + [1.0 / np.tanh(H_OVER_KB_K_PER_THZ * nu0 / (2 * t)) for t in TEMPS[1:]])
    want = (coth / nu0)[:, None, None] * np.array([1.0, 1, 1, 0, 0, 0])
    err = np.abs(got - want).max() / np.abs(want).max()
    print(f"Einstein identity through the kernel, 4096 q x 24 modes: {err:.2e}")
    assert err <= 1e-12


@pytest.fixture(scope="module")
def model030():
    return phonon_cells.model030()


def test_device_path_matches_spec_path(model030):
    ph = phonon_cells.limno2_222(model030)
    mesh = (20, 20, 20)  # 8 000 q: two eigh chunks of at most 4 096
    assert 20**3 > ph.eigh_batch
    d = ph.dynamical_matrices(np.zeros((2, 3)))
    e = torch.linalg.eigh(d)[1]
    print("eigh eigenvectors on the device: strides", e.stride(), "; e.mT contiguous:", e.mT.is_contiguous())
    got = ph.thermal_displacement_matrices(mesh, TEMPS)
    again = ph.thermal_displacement_matrices(mesh, TEMPS)
    spec = phonon_cells.spec_phonons(ph.force_constants, ph.cell)
    want = spec.thermal_displacement_matrices(mesh, TEMPS)
    scale = np.abs(want["cartesian"]).max()
    err = np.abs(got["cartesian"] - want["cartesian"]).max() / scale
    err_cif = np.abs(got["cif"] - want["cif"]).max() / np.abs(want["cif"]).max()
    print(f"LiMnO2 2x2x2 device force constants, 20^3 mesh, 31 temperatures: device vs specification path "
          f"{err:.2e} (cif {err_cif:.2e}) of max|U| = {scale:.3e} A^2; n_imaginary {got['n_imaginary']}; "
          f"U diagonals at 300 K (A^2):\n{np.diagonal(got['cartesian'][6], axis1=1, axis2=2)}")
    assert err <= 1e-9 and err_cif <= 1e-9
    assert got["n_imaginary"] == want["n_imaginary"]
    assert np.array_equal(got["cartesian"], again["cartesian"])


def test_fcc_cu(model030):
    ph = model030.phonons(CU, [4, 4, 4])
    fc = ph.force_constants[0]  # [N, 3, 3]
    sc = ph.cell
    # the noise of the unsymmetrised force constants: Phi(0, j) against its transpose and against Phi(0, -j) (the
    # atom at -r_j; fcc has inversion symmetry), relative to max|Phi|
    d = (-sc.frac)[:, None, :] - sc.frac[None, :, :]
    inv = np.argmax(np.all(np.abs(d - np.round(d)) < 1e-8, axis=2), axis=1)
    scale = np.abs(fc).max()
    noise = max(np.abs(fc - fc.transpose(0, 2, 1)).max(), np.abs(fc - fc[inv]).max()) / scale
    recip = np.linalg.inv(CU[2]).T
    unit = recip / np.linalg.norm(recip, axis=1)[:, None]
    print(f"fcc Cu 4x4x4: force-constant noise {noise:.2e} of max|Phi| = {scale:.3f} eV/A^2, asr_correction "
          f"{ph.asr_correction:.2e} eV/A^2")
    for n in (8, 16, 24):
        out = ph.thermal_displacement_matrices((n, n, n), [300.0])
        u = out["cartesian"][0, 0]
        u_iso = np.trace(u) / 3
        aniso = np.abs(u - u_iso * np.eye(3)).max() / u_iso
        cif_err = np.abs(out["cif"][0, 0] - u_iso * unit @ unit.T).max() / u_iso
        print(f"  mesh {n}^3, 300 K: U =\n{u}\n  U_iso {u_iso:.6f} A^2, anisotropy {aniso:.2e}, cif vs u cos(a*_i, a*_j) "
              f"{cif_err:.2e}, n_imaginary {out['n_imaginary']}")
        assert np.isfinite(u).all() and u_iso > 0
        # U goes as 1 / nu^2, i.e. as the inverse of D's eigenvalues: a relative perturbation of Phi moves U by about
        # as much, more where modes are soft.  Measured on an H100 with the 0.3.0 weights: noise 2.4e-3, anisotropy
        # 7.2e-6, 3.9e-5 and 1.2e-3 on 8^3, 16^3 and 24^3 (Cu shows imaginary modes at this lattice constant, so U is
        # not compared with experiment)
        tol = max(4 * noise, 1e-9)
        assert aniso <= tol and cif_err <= tol
