"""CPU (fp64): the three-phonon specifications on the shapes of tests/test_three_phonon_shapes_gpu.py.

* the planted axis-reversed split of the mesh indices (``axes_reversed``, tests/three_phonon_kernels.py) gives exactly
  the true specification on a cubic mesh, and P, Gamma, the collision rows and the spectrum far from it on every
  non-cubic mesh of the device table: the evidence that those rows catch a swapped axis that the cubic ones cannot;
* the specification of ``chg_imag_self_energy`` against a plain loop on (4, 3, 5) at 9 temperatures with a forced
  tetrahedron diagonal other than 0;
* the specifications on frequencies quantised to 0.25 THz (corner values tied, and on the points): every output is
  finite."""
import numpy as np
import pytest
import torch

from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, tetrahedra
from lbte_kernels import LbteSpecKernels
from spectral_function_kernels import SpectralFunctionSpecKernels
from test_three_phonon_shapes_gpu import CASES, T9, T17
from test_three_phonon_spec import _limno2_spec_ph, _loop_gamma, _spring_phonons

CUT = THERMAL_CUTOFF_THZ
f64 = torch.float64
NON_CUBIC = sorted({c[2] for c in CASES.values() if len(set(c[2])) > 1})


@pytest.fixture(scope="module")
def limno2(weights030):
    """LiMnO2 2x1x1 (24 bands) with a random symmetric fc3, on the specification path, and its kernel arguments."""
    ph = _limno2_spec_ph(weights030, seed=6)
    frac = torch.as_tensor(np.ascontiguousarray(ph.cell.prim_frac, dtype=np.float64))
    return ph, (ph._fc3, ph._img_ptr, ph._img_vec, ph._s2p, ph._inv_sqrt_m, frac)


def _outputs(k, k_sf, args, mesh, nu, e, tets, target, q1, temps, points, p=None):
    """(P, Gamma, collision rows, spectrum) of the specification kernels k (``LbteSpecKernels``) and k_sf
    (``SpectralFunctionSpecKernels``); the consumers take ``p`` when given, else the P computed here."""
    n_mesh, nb = nu.shape
    pk = torch.empty(len(q1), nb, nb, nb, dtype=f64)
    k.phonon_interaction(*args, mesh, nu, e, target, q1, CUT, pk)
    p = pk if p is None else p
    omega = nu[target].contiguous()
    gamma = torch.zeros(len(temps), nb, dtype=f64)
    rows = torch.zeros(4, len(temps), nb, n_mesh, nb, dtype=f64)
    se = torch.zeros(len(temps), nb, len(points), dtype=f64)
    k.imag_self_energy(nu, mesh, tets, target, omega, q1, p, temps, CUT, gamma)
    k.collision_rows(nu, mesh, tets, target, omega, q1, p, temps, CUT, rows)
    k_sf.self_energy_spectrum(nu, mesh, tets, target, points, q1, p, temps, CUT, se)
    return pk, gamma, rows, se


@pytest.mark.parametrize("mesh", [(3, 3, 3)] + NON_CUBIC, ids=lambda m: "x".join(map(str, m)))
def test_axis_reversal_caught_only_off_cubic(limno2, mesh):
    ph, args = limno2
    mesh_t, nu, e, _, tets, _ = ph._three_phonon_mesh(mesh, None)
    n_mesh = nu.shape[0]
    target = n_mesh - 2
    q1 = torch.arange(0, n_mesh, max(1, n_mesh // 12), dtype=torch.int32)
    temps = torch.tensor(T9, dtype=f64)
    points = torch.linspace(0.0, 2 * float(nu.max()), 33, dtype=f64)
    true = _outputs(LbteSpecKernels(), SpectralFunctionSpecKernels(), args, mesh_t, nu, e, tets, target, q1, temps,
                    points)
    # the consumers get the true P, so that each of them is shown to see the split on its own
    bad = _outputs(LbteSpecKernels(axes_reversed=True), SpectralFunctionSpecKernels(axes_reversed=True), args, mesh_t,
                   nu, e, tets, target, q1, temps, points, p=true[0])
    names = ("P", "Gamma", "rows", "spectrum")
    if len(set(mesh)) == 1:
        for name, a, b in zip(names, true, bad):
            assert torch.equal(a, b), name
        print(f"{mesh}: the axis-reversed split equals the specification bit for bit")
        return
    diff = {n: float((a - b).abs().max() / a.abs().max()) for n, a, b in zip(names, true, bad)}
    print(f"{mesh}, target {target}: the axis-reversed split differs from the specification by "
          + ", ".join(f"{k} {v:.2e}" for k, v in diff.items()) + " of max")
    # the device tolerances are 1e-12 (P), 1e-11 (Gamma) and 5e-15 (rows, spectrum)
    assert min(diff.values()) >= 1e-3


def test_imag_self_energy_against_loop_non_cubic():
    ph, _ = _spring_phonons()
    mesh = (4, 3, 5)
    mesh_t, nu, _, _, _, _ = ph._three_phonon_mesh(mesh, None)
    tets = torch.as_tensor(tetrahedra(mesh, ph.cell.prim_lattice, diagonal=2))
    assert not torch.equal(tets, torch.as_tensor(tetrahedra(mesh, ph.cell.prim_lattice)))
    rng = np.random.default_rng(2)
    p = torch.as_tensor(rng.random((60, 3, 3, 3)) * 1e-6)
    t = torch.tensor(T9, dtype=f64)
    target = 28  # mesh coordinates (1, 2, 3)
    gamma = torch.zeros(len(T9), 3, dtype=f64)
    ph.kernels.imag_self_energy(nu, mesh_t, tets, target, nu[target].contiguous(), torch.arange(60, dtype=torch.int32),
                                p, t, CUT, gamma)
    want = _loop_gamma(nu.numpy(), mesh_t, tets.numpy(), target, p.numpy(), T9)
    err = np.abs(gamma.numpy() - want).max() / np.abs(want).max()
    print(f"spring crystal {mesh}, diagonal 2, 9 temperatures: imag_self_energy spec vs plain loop {err:.2e}")
    assert np.abs(want).max() > 0 and err <= 1e-13


def test_spec_finite_on_quantised_frequencies(limno2):
    ph, args = limno2
    mesh = (4, 3, 5)
    mesh_t, nu, e, _, tets, _ = ph._three_phonon_mesh(mesh, None)
    nu = torch.round(nu * 4) / 4
    nu[0::3, 3], nu[1::3, 3], nu[2::3, 3] = CUT, 0.0, -0.25  # at, and below, the cutoff
    nu = torch.sort(nu, dim=1)[0].contiguous()
    q1 = torch.arange(0, 60, 5, dtype=torch.int32)
    points = torch.arange(33, dtype=f64) * 1.25
    out = _outputs(LbteSpecKernels(), SpectralFunctionSpecKernels(), args, mesh_t, nu, e, tets, 28, q1,
                   torch.tensor(T17, dtype=f64), points)
    for name, x in zip(("P", "Gamma", "rows", "spectrum"), out):
        assert bool(torch.isfinite(x).all()) and bool(x.any()), name
