"""-m gpu: isotope and boundary scattering on the device (Phonons.isotope_linewidths and the options of the thermal
conductivities).

* ``chg_isotope_scattering`` against its fp64 specification (tests/isotope_kernels.py, run with torch on the same
  device) on random unitary eigenvectors, random mass variances with zeros and frequencies with negative and
  sub-cutoff values: 24 bands on 8^3 with 37 targets and 93 bands on 4^3; two calls bitwise equal, targets split over
  calls bitwise equal to one call;
* the completeness identity against ``chg_tetrahedron_dos``;
* on the device fc3 of LiMnO2 2x2x2, ``isotope_linewidths`` on 8^3 and the three conductivities on 6^3 with both
  options against the specification path, and bitwise the calls without options when the options are None."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, Phonons, gamma_mesh, tetrahedra
from isotope_kernels import IsotopeSpecKernels

pytestmark = pytest.mark.gpu
CUT = THERMAL_CUTOFF_THZ
# illustrative mass variances of LiMnO2's atoms (Li, Mn, O); not natural-abundance data
G_LIMNO2 = [1.5e-3, 1.5e-3, 0.0, 0.0, 3.4e-5, 3.4e-5, 3.4e-5, 3.4e-5]


def _random_inputs(mesh, nb, n_target, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    f64, dev = torch.float64, "cuda"
    n_q = mesh[0] * mesh[1] * mesh[2]
    nu = torch.rand(n_q, nb, generator=g, device=dev, dtype=f64) * 23.0 - 3.0
    nu[::3, 1] = 5e-4
    nu[1::3, 1] = CUT
    nu = torch.sort(nu, dim=1)[0].contiguous()
    a = torch.complex(torch.randn(n_q, nb, nb, generator=g, device=dev, dtype=f64),
                      torch.randn(n_q, nb, nb, generator=g, device=dev, dtype=f64))
    e = torch.linalg.qr(a)[0].mT.contiguous()
    mv = torch.rand(nb // 3, generator=g, device=dev, dtype=f64) * 2e-3
    mv[::4] = 0.0
    targets = torch.randint(0, n_q, (n_target,), generator=g, device=dev, dtype=torch.int32)
    targets[0], targets[-1] = 0, n_q - 1
    omega = nu[targets.long()].clone()
    omega[1::5] = torch.rand(omega[1::5].shape, generator=g, device=dev, dtype=f64) * 20.0  # off the band frequencies
    omega[2, :4] = torch.tensor([-1.0, 0.0, 5e-4, CUT], dtype=f64)
    tets = torch.as_tensor(tetrahedra(mesh, np.eye(3))).to(dev)
    return nu, e, mv, targets, omega.contiguous(), tets


@pytest.mark.parametrize("mesh,nb,n_target", [((8, 8, 8), 24, 37), ((4, 4, 4), 93, 9)])
def test_kernel_matches_spec(mesh, nb, n_target):
    from chgnet_b200._lib import CudaKernels

    nu, e, mv, targets, omega, tets = _random_inputs(mesh, nb, n_target, seed=nb + n_target)
    kern, spec = CudaKernels("cuda"), IsotopeSpecKernels()

    def run(k, step=n_target):
        out = torch.full((n_target, nb), float("nan"), dtype=torch.float64, device="cuda")
        for s in range(0, n_target, step):
            k.isotope_scattering(nu, mesh, tets, e, mv, targets[s : s + step], omega[s : s + step], CUT,
                                 out[s : s + step])
        return out

    got, again, want = run(kern), run(kern), run(spec)
    split = run(kern, 5)
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    print(f"{nb} bands on {mesh}, {n_target} targets: kernel vs specification {err:.2e} of max|Gamma| {scale:.3e}; "
          f"bitwise reproducible; 5-target calls bitwise equal to one call")
    assert torch.equal(got, again) and torch.equal(split, got)
    assert scale > 0 and torch.all(got[2, :3] == 0) and got[2, 3] != 0 and torch.all(got[omega < CUT] == 0)
    assert err <= 5e-15


def test_completeness_on_device():
    from chgnet_b200._lib import CudaKernels

    mesh, nb = (6, 5, 4), 12
    nu, e, mv, targets, _, tets = _random_inputs(mesh, nb, 4, seed=3)
    kern = CudaKernels("cuda")
    n_q = nu.shape[0]
    proj = torch.where((nu >= CUT)[..., None], (e.abs() ** 2).view(n_q, nb, nb // 3, 3).sum(-1), 0.0).contiguous()
    w0s = torch.tensor([2.0, 7.5, 13.0, 18.5], dtype=torch.float64, device="cuda")
    dos, idos = torch.empty_like(w0s), torch.empty_like(w0s)
    pdos = torch.empty(nb // 3, len(w0s), dtype=torch.float64, device="cuda")
    kern.tetrahedron_dos(nu, mesh, tets, w0s, dos, idos, proj, pdos)
    worst = 0.0
    for i, w0 in enumerate(w0s.tolist()):
        om = torch.full((len(targets), nb), w0, dtype=torch.float64, device="cuda")
        gamma = torch.empty_like(om)
        kern.isotope_scattering(nu, mesh, tets, e, mv, targets, om, CUT, gamma)
        want = np.pi / 4 * w0**2 * float((mv * pdos[:, i]).sum())
        worst = max(worst, float((gamma.sum(1) - want).abs().max()) / want)
    print(f"12 bands on {mesh}: sum_l Gamma_l(w0) vs (pi/4) w0^2 sum g pdos (chg_tetrahedron_dos) {worst:.2e}")
    assert worst <= 1e-13


@pytest.fixture(scope="module")
def limno2_fc3():
    model = phonon_cells.model030()
    return model.phonons(graphgen.limno2_structure(), [2, 2, 2], third_order=True)


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def test_isotope_linewidths_device_vs_spec(limno2_fc3):
    ph = limno2_fc3
    spec = Phonons(ph.force_constants, ph.cell, device="cuda", kernels=IsotopeSpecKernels())
    mesh = (8, 8, 8)
    q = gamma_mesh(mesh)[::7]
    got, want = ph.isotope_linewidths(mesh, q, G_LIMNO2), spec.isotope_linewidths(mesh, q, G_LIMNO2)
    err = _rel(got["isotope_linewidths"], want["isotope_linewidths"])
    print(f"LiMnO2 2x2x2 on 8^3, {len(q)} q: isotope_linewidths device vs specification path {err:.2e}; max "
          f"{np.abs(got['isotope_linewidths']).max():.3e} THz")
    assert np.abs(got["frequencies"] - want["frequencies"]).max() <= 1e-9
    # the two paths diagonalise D from different (rounding-equal) D(q) kernels: measured 7.3e-13 on an H100
    assert err <= 5e-12


def test_conductivities_device_vs_spec(limno2_fc3):
    ph = limno2_fc3
    spec = Phonons(ph.force_constants, ph.cell, fc3=ph.force_constants3, device="cuda", kernels=IsotopeSpecKernels())
    mesh, temps = (6, 6, 6), [0.0, 300.0, 1000.0]
    opts = {"mass_variances": G_LIMNO2, "boundary_mfp": 0.5}
    report = []
    for name in ("thermal_conductivity", "thermal_conductivity_lbte", "thermal_conductivity_wigner"):
        got, want = getattr(ph, name)(mesh, temps, **opts), getattr(spec, name)(mesh, temps, **opts)
        plain = getattr(ph, name)(mesh, temps)
        none = getattr(ph, name)(mesh, temps, mass_variances=None, boundary_mfp=None)
        assert set(none) == set(plain)
        for k in plain:
            assert np.array_equal(none[k], plain[k], equal_nan=True), (name, k)
        err = _rel(got["kappa"], want["kappa"])
        err_iso = _rel(got["isotope_linewidths"], want["isotope_linewidths"])
        report.append(f"{name} {err:.2e} (isotope {err_iso:.2e}; 300 K diagonal {np.diag(got['kappa'][1])} vs "
                      f"{np.diag(plain['kappa'][1])} without)")
        # measured <= 5.8e-14 for kappa and <= 3.9e-13 for Gamma^iso on an H100
        assert np.all(got["kappa"][0] == 0) and err <= 1e-12 and err_iso <= 5e-12
        if name == "thermal_conductivity":
            rta = got
        elif name == "thermal_conductivity_lbte":
            assert np.array_equal(got["kappa_rta"], rta["kappa"])
        else:
            assert np.array_equal(got["kappa_p"], rta["kappa"])
    print("LiMnO2 2x2x2 on 6^3 at 0, 300, 1000 K with isotopes and L = 0.5 um, device vs specification path: "
          + "; ".join(report))
