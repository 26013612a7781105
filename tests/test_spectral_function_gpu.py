"""-m gpu: the self-energy spectrum and the phonon spectral functions on the device (Phonons.spectral_function).

* ``chg_self_energy_spectrum`` at the target's own band frequencies against ``chg_imag_self_energy`` (the diagonal
  band = point);
* ``chg_self_energy_spectrum`` against its fp64 specification (tests/spectral_function_kernels.py, run with torch on
  the same device) on random P and frequencies with negative and sub-cutoff values on a 201-point grid: 24 bands on 8^3
  and 93 bands (31 atoms) on 4^3; two calls bitwise equal;
* on the device fc3 of LiMnO2 2x2x2, ``spectral_function`` on 6^3 at 0, 300 and 1 000 K against the specification
  path."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, Phonons
from spectral_function_kernels import SpectralFunctionSpecKernels
from test_three_phonon_gpu import _random_case

pytestmark = pytest.mark.gpu
CUT = THERMAL_CUTOFF_THZ


def _random_p(nu, mesh, target, seed):
    """Random P [N, 3n, 3n, 3n] (about 1e-6 eV^2), 0 wherever a mode of the triplet is below the cutoff."""
    n_mesh, nb = nu.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    keep = (nu >= CUT)[target][:, None, None] & (nu >= CUT)[:, None, :, None]
    p = torch.rand(n_mesh, nb, nb, nb, generator=g, device="cuda", dtype=torch.float64) * 1e-6
    i2 = [np.ravel_multi_index(tuple((np.array(np.unravel_index(target, mesh)) - np.array(np.unravel_index(i, mesh)))
                                     % mesh), mesh) for i in range(n_mesh)]
    return torch.where(keep & (nu[torch.as_tensor(i2, device="cuda")] >= CUT)[:, None, None, :], p, 0.0).contiguous()


TEMPS = [0.0, 300.0, 1000.0]


def test_kernel_matches_imag_self_energy():
    from chgnet_b200._lib import CudaKernels

    mesh, target = (8, 8, 8), 77
    _, nu, _, tets = _random_case(8, (2, 2, 2), mesh, seed=16)
    nb, n_mesh = nu.shape[1], int(np.prod(mesh))
    p = _random_p(nu, mesh, target, 3)
    temps = torch.tensor(TEMPS, dtype=torch.float64, device="cuda")
    omega = nu[target].contiguous()
    kern = CudaKernels("cuda")
    q1 = torch.arange(n_mesh, dtype=torch.int32, device="cuda")
    want = torch.zeros(3, nb, dtype=torch.float64, device="cuda")
    got = torch.zeros(3, nb, nb, dtype=torch.float64, device="cuda")
    for s in range(0, n_mesh, 128):
        kern.imag_self_energy(nu, mesh, tets, target, omega, q1[s : s + 128], p[s : s + 128], temps, CUT, want)
        kern.self_energy_spectrum(nu, mesh, tets, target, omega, q1[s : s + 128], p[s : s + 128], temps, CUT, got)
    diag = got.diagonal(dim1=1, dim2=2)
    scale = want.abs().max()
    err = float((diag - want).abs().max() / scale)
    print(f"24 bands, 8^3, target {target}: self_energy_spectrum at the band frequencies vs imag_self_energy "
          f"{err:.2e} of max|Gamma| {float(scale):.3e}")
    assert scale > 0 and err <= 1e-14


@pytest.mark.parametrize("n_prim,cells,mesh,target,spec_q1", [
    (8, (2, 2, 2), (8, 8, 8), 77, 48),
    (31, (2, 1, 1), (4, 4, 4), 21, 6),
])
def test_kernel_matches_spec(n_prim, cells, mesh, target, spec_q1):
    from chgnet_b200._lib import CudaKernels

    _, nu, _, tets = _random_case(n_prim, cells, mesh, seed=n_prim + mesh[0] + 2)
    nb, n_mesh = 3 * n_prim, int(np.prod(mesh))
    p = _random_p(nu, mesh, target, 7)
    temps = torch.tensor(TEMPS, dtype=torch.float64, device="cuda")
    grid = torch.arange(201, dtype=torch.float64, device="cuda") * (float(2 * nu.max()) / 200)
    kern, spec = CudaKernels("cuda"), SpectralFunctionSpecKernels()

    def run(k, q1s):
        out = torch.zeros(len(temps), nb, len(grid), dtype=torch.float64, device="cuda")
        k.self_energy_spectrum(nu, mesh, tets, target, grid, q1s, p[q1s.long()].contiguous(), temps, CUT, out)
        return out

    q1 = torch.arange(n_mesh, dtype=torch.int32, device="cuda")
    a, b = run(kern, q1), run(kern, q1)
    assert torch.equal(a, b)
    sub = q1[torch.linspace(0, n_mesh - 1, spec_q1, device="cuda").long()]
    got, want = run(kern, sub), run(spec, sub)
    scale = want.abs().max()
    err = float((got - want).abs().max() / scale)
    print(f"{nb} bands, {mesh[0]}^3, target {target}, 201 points: {n_mesh} q1 bitwise reproducible; on {spec_q1} q1 "
          f"Gamma(w) {err:.2e} of max|Gamma| {float(scale):.3e} against the specification")
    assert scale > 0 and err <= 5e-15


@pytest.fixture(scope="module")
def limno2_fc3():
    model = phonon_cells.model030()
    return model.phonons(graphgen.limno2_structure(), [2, 2, 2], third_order=True)


def test_device_path_matches_spec_path(limno2_fc3):
    ph = limno2_fc3
    spec = Phonons(ph.force_constants, ph.cell, fc3=ph.force_constants3, device="cuda",
                   kernels=SpectralFunctionSpecKernels())
    mesh = (6, 6, 6)
    q = np.array([[1 / 3, 1 / 6, 0.5], [0.0, 0.0, 0.0]])
    got, want = ph.spectral_function(mesh, q, TEMPS), spec.spectral_function(mesh, q, TEMPS)
    errs = {k: float(np.abs(got[k] - want[k]).max() / np.abs(want[k]).max())
            for k in ("gamma", "delta", "spectral_function", "frequency_shifts")}
    lw = ph.linewidths(mesh, q, TEMPS)["linewidths"]
    print(f"LiMnO2 2x2x2 on 6^3 at 0, 300, 1000 K: device vs specification path {errs}; largest shift at 300 K "
          f"{np.abs(got['frequency_shifts'][1]).max():.4f} THz, largest linewidth {lw[1].max():.4f} THz")
    # the grids come from each path's highest mesh frequency, which agree to a few ulps
    assert np.abs(got["self_energy_points"] - want["self_energy_points"]).max() <= 1e-14 * want["self_energy_points"][-1]
    assert np.all(got["gamma"][0] >= 0) and got["n_imaginary"] == want["n_imaginary"]
    # measured on an H100 in two sessions: Gamma 1.7e-11 and 2.4e-11, Delta 1.0e-11 and 1.4e-11, shifts 1.1e-12 and
    # 2.0e-12, A 3.1e-10 and 3.8e-10 (A amplifies them near its peaks)
    assert errs["gamma"] <= 1e-10 and errs["delta"] <= 1e-10 and errs["frequency_shifts"] <= 1e-10
    assert errs["spectral_function"] <= 3e-9
