"""-m gpu: the collision-matrix rows and the LBTE thermal conductivity on the device (Phonons.thermal_conductivity_lbte).

* ``chg_collision_rows`` against its fp64 specification (tests/lbte_kernels.py, run with torch on the same device) on
  random unitary eigenvectors, random P and frequencies with negative and sub-cutoff values: 24 bands on 8^3 and 93
  bands (31 atoms) on 4^3; two calls bitwise equal;
* on the device fc3 of LiMnO2 2x2x2, ``thermal_conductivity_lbte`` on 4^3 and 6^3 at 0, 300 and 1 000 K against the
  specification path."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, Phonons
from lbte_kernels import LbteSpecKernels
from test_three_phonon_gpu import _random_case

pytestmark = pytest.mark.gpu
CUT = THERMAL_CUTOFF_THZ


@pytest.mark.parametrize("n_prim,cells,mesh,target,spec_q1", [
    (8, (2, 2, 2), (8, 8, 8), 77, 48),
    (31, (2, 1, 1), (4, 4, 4), 21, 6),
])
def test_collision_rows_match_spec(n_prim, cells, mesh, target, spec_q1):
    from chgnet_b200._lib import CudaKernels

    _, nu, _, tets = _random_case(n_prim, cells, mesh, seed=n_prim + mesh[0] + 1)
    nb, n_mesh = 3 * n_prim, int(np.prod(mesh))
    g = torch.Generator(device="cuda").manual_seed(7)
    keep = ((nu >= CUT)[target][:, None, None] & (nu >= CUT)[:, None, :, None])  # P = 0 below the cutoff
    p = torch.rand(n_mesh, nb, nb, nb, generator=g, device="cuda", dtype=torch.float64) * 1e-6
    i2 = [np.ravel_multi_index(tuple((np.array(np.unravel_index(target, mesh)) - np.array(np.unravel_index(i, mesh)))
                                     % mesh), mesh) for i in range(n_mesh)]
    p = torch.where(keep & (nu[torch.as_tensor(i2, device="cuda")] >= CUT)[:, None, None, :], p, 0.0).contiguous()
    temps = torch.tensor([0.0, 50.0, 300.0, 1000.0, 1e4], dtype=torch.float64, device="cuda")
    omega = nu[target].contiguous()
    kern, spec = CudaKernels("cuda"), LbteSpecKernels()

    def run(k, q1s):
        out = torch.zeros(4, len(temps), nb, n_mesh, nb, dtype=torch.float64, device="cuda")
        k.collision_rows(nu, mesh, tets, target, omega, q1s, p[q1s.long()].contiguous(), temps, CUT, out)
        return out

    q1 = torch.arange(n_mesh, dtype=torch.int32, device="cuda")
    a, b = run(kern, q1), run(kern, q1)
    assert torch.equal(a, b)
    sub = q1[torch.linspace(0, n_mesh - 1, spec_q1, device="cuda").long()]
    got, want = run(kern, sub), run(spec, sub)
    scale = want.abs().max()
    err = float((got - want).abs().max() / scale)
    print(f"{nb} bands, {mesh[0]}^3, target {target}: {n_mesh} q1 bitwise reproducible; on {spec_q1} q1 collision rows "
          f"{err:.2e} of max|R| {float(scale):.3e} against the specification")
    assert scale > 0 and err <= 5e-15


@pytest.fixture(scope="module")
def limno2_fc3():
    model = phonon_cells.model030()
    return model.phonons(graphgen.limno2_structure(), [2, 2, 2], third_order=True)


# kappa's tolerance: on 4^3 this unrelaxed cell's matrix is ill-conditioned (kappa_LBTE is 8x kappa_RTA along x, from
# small eigenvalues), and it amplifies the 1e-12-level agreement of the linewidths (section 12.7) to 3.6e-10 - 8.8e-10
@pytest.mark.parametrize("mesh,tol", [((4, 4, 4), 2e-9), ((6, 6, 6), 1e-12)])
def test_device_path_matches_spec_path(limno2_fc3, mesh, tol):
    ph = limno2_fc3
    spec = Phonons(ph.force_constants, ph.cell, fc3=ph.force_constants3, device="cuda", kernels=LbteSpecKernels())
    temps = [0.0, 300.0, 1000.0]
    got, want = ph.thermal_conductivity_lbte(mesh, temps), spec.thermal_conductivity_lbte(mesh, temps)
    err = np.abs(got["kappa"] - want["kappa"]).max() / np.abs(want["kappa"]).max()
    err_rta = np.abs(got["kappa_rta"] - want["kappa_rta"]).max() / np.abs(want["kappa_rta"]).max()
    print(f"LiMnO2 2x2x2 LBTE on {mesh[0]}^3 at 0, 300, 1000 K: device vs specification path kappa {err:.2e}, kappa_rta "
          f"{err_rta:.2e}; kappa(300 K) diagonal {np.diag(got['kappa'][1])}, RTA {np.diag(got['kappa_rta'][1])} "
          f"W/(m K); dropped {got['n_dropped'].tolist()}, min eigenvalue {got['min_eigenvalue'].tolist()} 1/ps")
    assert np.all(got["kappa"][0] == 0)
    assert err <= tol and err_rta <= 1e-9
    assert list(got["n_dropped"]) == list(want["n_dropped"])
    assert list(got["n_zero_linewidth"]) == list(want["n_zero_linewidth"])
