"""-m gpu: two-phonon joint densities of states on the device (Phonons.joint_dos, Phonons.phase_space).

* ``chg_joint_dos`` against its fp64 specification (oracle/phonons.py, run with torch on the same device) on random
  ascending frequencies with negative values, values below and on the cutoff: 24 bands on a 16^3 mesh with 256
  targets at their own 24 mode frequencies (n_t = 0 and n_t = 31), 93 bands (31 atoms) on 4^3 with a 201-point grid,
  and frequencies on a coarse grid (tied corner values, frequency points on corner values); bitwise reproducible;
* the device force constants of LiMnO2 2x2x2: ``joint_dos`` and ``phase_space`` on a 10^3 mesh against the
  specification path on the same force constants."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, Phonons, tetrahedra
from oracle.phonons import PhononSpecKernels

pytestmark = pytest.mark.gpu

TEMPS = np.linspace(0.0, 1500.0, 31)


def _random_freqs(n_q, n_band, seed, grid=None):
    """[n_q, n_band] ascending frequencies on the device in [-3, 20) THz, with 0, 5e-4, the cutoff and -1e-2 among
    them; ``grid`` rounds them to multiples of that step (ties everywhere)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    nu = torch.rand(n_q, n_band, generator=g, device="cuda", dtype=torch.float64) * 23.0 - 3.0
    nu[:, 0] = 0.0
    nu[::3, 1] = 5e-4
    nu[1::3, 1] = THERMAL_CUTOFF_THZ
    nu[2::3, 1] = -1e-2
    if grid is not None:
        nu = torch.round(nu / grid) * grid
    return torch.sort(nu, dim=1)[0].contiguous()


def _compare(case, nu, mesh, targets, omega, temps, spec_every=1):
    from chgnet_b200._lib import CudaKernels

    tets = torch.as_tensor(tetrahedra(mesh, np.eye(3))).cuda()
    tg = torch.as_tensor(np.asarray(targets, dtype=np.int32)).cuda()
    t = None if temps is None else torch.as_tensor(temps).cuda()
    n_slots = 1 + (0 if temps is None else len(temps))
    kern = CudaKernels("cuda")

    def run(k, tg, omega):
        out = torch.empty(len(tg), n_slots, 2, omega.shape[1], dtype=torch.float64, device="cuda")
        k.joint_dos(nu, mesh, tets, tg, omega, t, THERMAL_CUTOFF_THZ, out)
        return out

    got, again = run(kern, tg, omega), run(kern, tg, omega)
    spec = PhononSpecKernels()
    spec.jdos_chunk_items = 1 << 20
    sub = slice(None, None, spec_every)
    want = run(spec, tg[sub].contiguous(), omega[sub].contiguous())
    scale = float(want.abs().max())
    err = float((got[sub] - want).abs().max()) / scale
    print(f"{case}: max|kernel - spec| / max = {err:.2e} (max {scale:.3e} 1/THz, {len(want)} of {len(tg)} targets "
          f"checked)")
    assert err <= 1e-10
    assert torch.equal(got, again)
    return got


@pytest.mark.parametrize("n_t", [0, 31])
def test_kernel_matches_spec_24_bands_16_cubed(n_t):
    mesh, nb = (16, 16, 16), 24
    nu = _random_freqs(16**3, nb, seed=7 + n_t)
    targets = np.random.default_rng(3).choice(16**3, 256, replace=False)
    targets[0] = 0
    omega = nu[torch.as_tensor(targets).cuda().long()].contiguous()  # phase-space layout: each target's own modes
    _compare(f"24 bands, 16^3, 256 targets x 24 points, n_t = {n_t}", nu, mesh, targets, omega,
             TEMPS if n_t else None, spec_every=8)


def test_kernel_matches_spec_93_bands():
    mesh, nb = (4, 4, 4), 93
    nu = _random_freqs(64, nb, seed=31)
    omega = torch.linspace(-5.0, 40.0, 201, dtype=torch.float64, device="cuda")[None].expand(6, -1).contiguous()
    _compare("93 bands (31 atoms), 4^3, 6 targets x 201 points, 3 temperatures", nu, mesh, [0, 1, 5, 21, 42, 63], omega,
             np.array([0.0, 300.0, 1000.0]))


def test_kernel_matches_spec_ties_and_vertices():
    mesh, nb = (6, 5, 4), 6
    nu = _random_freqs(120, nb, seed=2, grid=0.5)
    omega = torch.arange(-8.0, 40.5, 0.5, dtype=torch.float64, device="cuda")[None].expand(10, -1).contiguous()
    _compare("6 bands on a 0.5 THz grid, 6x5x4, points on the grid, 31 temperatures", nu, mesh, np.arange(0, 120, 12),
             omega, TEMPS)


@pytest.fixture(scope="module")
def limno2_222():
    return phonon_cells.limno2_222(phonon_cells.model030())


def test_device_path_matches_spec_path(limno2_222):
    ph = limno2_222
    mesh = (10, 10, 10)
    spec = Phonons(ph.force_constants, ph.cell, device="cuda", kernels=PhononSpecKernels())
    spec.kernels.jdos_chunk_items = 1 << 20
    # away from Gamma: there the class-1 tetrahedra of l1 = l2 are flat to rounding and D2(1) at w = 0 is ~1/ulp
    q = np.array([[0.3, 0.3, 0.0], [0.5, 0.0, 0.0], [0.1, 0.2, 0.3], [-0.4, 0.5, 0.7]])
    got = ph.joint_dos(mesh, q, temperatures=TEMPS)
    # the default grid ends at twice the highest frequency, which the two D(q) builds give to a few ulp
    assert np.abs(got["frequency_points"] - spec.joint_dos(mesh, q[0])["frequency_points"]).max() <= 1e-12 * 40
    want = spec.joint_dos(mesh, q, got["frequency_points"], TEMPS)
    err = np.abs(got["jdos"] - want["jdos"]).max() / np.abs(want["jdos"]).max()
    err_w = np.abs(got["weighted_jdos"] - want["weighted_jdos"]).max() / np.abs(want["weighted_jdos"]).max()
    print(f"LiMnO2 2x2x2 device force constants, joint_dos on 10^3 at 4 q, 201 points, 31 T: device vs specification "
          f"path {err:.2e} (weighted {err_w:.2e}); n_imaginary {got['n_imaginary']}")
    assert err <= 1e-9 and err_w <= 1e-9
    assert got["n_imaginary"] == want["n_imaginary"]
    temps = [0.0, 300.0, 1000.0]
    got = ph.phase_space(mesh, temps)
    again = ph.phase_space(mesh, temps)
    want = spec.phase_space(mesh, temps)
    err = np.abs(got["jdos"] - want["jdos"]).max() / np.abs(want["jdos"]).max()
    err_w = np.abs(got["weighted_jdos"] - want["weighted_jdos"]).max() / np.abs(want["weighted_jdos"]).max()
    err_a = np.abs(got["average_weighted_jdos"] - want["average_weighted_jdos"]).max() / np.abs(
        want["average_weighted_jdos"]).max()
    print(f"LiMnO2 2x2x2, phase_space on 10^3 at 0, 300, 1000 K: device vs specification path {err:.2e} (weighted "
          f"{err_w:.2e}, averages {err_a:.2e}); average_jdos {got['average_jdos']}, average_weighted_jdos "
          f"{got['average_weighted_jdos'].tolist()}; n_imaginary {got['n_imaginary']}")
    assert err <= 1e-9 and err_w <= 1e-9 and err_a <= 1e-9
    assert got["n_imaginary"] == want["n_imaginary"]
    assert np.array_equal(got["weighted_jdos"], again["weighted_jdos"])
