"""-m gpu: third-order force constants, three-phonon interaction strengths and linewidths on the device
(Phonons.linewidths, Phonons.thermal_conductivity).

* ``chg_phonon_interaction`` and ``chg_imag_self_energy`` against their fp64 specifications (tests/three_phonon_kernels.py,
  run with torch on the same device) on random unitary eigenvectors, random fc3 and frequencies with negative and
  sub-cutoff values: 24 bands on 8^3 and 12^3, 93 bands (31 atoms) on 4^3; two calls bitwise equal;
* the device fc3 of LiMnO2 2x2x2 (0.3.0 weights) against central differences of the fp64 oracle's Hessian-vector
  products at the same h, on a slice of (k, a) and columns, and its translational-sum residual;
* on that fc3, ``linewidths`` at several q and ``thermal_conductivity`` on 6^3 against the specification path."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, Phonons, make_supercell, tetrahedra
from oracle.hessian import oracle_hvp
from three_phonon_kernels import ThreePhononSpecKernels

pytestmark = pytest.mark.gpu
CUT = THERMAL_CUTOFF_THZ


def _random_case(n_prim, cells, mesh, seed):
    """A random cell of n_prim atoms on the supercell ``cells``, a random fc3, and random frequencies [N, 3n] (with 0,
    5e-4, the cutoff and -1e-2 among them) and unitary mode-major eigenvectors on ``mesh``, all on the device."""
    rng = np.random.default_rng(seed)
    lat = np.diag([4.0, 4.5, 5.0]) + 0.3 * rng.random((3, 3))
    sc = make_supercell(np.full(n_prim, 14), rng.random((n_prim, 3)), lat, cells)
    n, nb, n_q = len(sc.z), 3 * n_prim, int(np.prod(mesh))
    g = torch.Generator(device="cuda").manual_seed(seed)
    fc3 = torch.randn(n_prim, n, n, 3, 3, 3, generator=g, device="cuda", dtype=torch.float64)
    nu = torch.rand(n_q, nb, generator=g, device="cuda", dtype=torch.float64) * 23.0 - 3.0
    nu[:, 0] = 0.0
    nu[::3, 1] = 5e-4
    nu[1::3, 1] = CUT
    nu[2::3, 1] = -1e-2
    nu = torch.sort(nu, dim=1)[0].contiguous()
    a = torch.randn(n_q, nb, nb, generator=g, device="cuda", dtype=torch.float64) + 1j * torch.randn(
        n_q, nb, nb, generator=g, device="cuda", dtype=torch.float64)
    e = torch.linalg.qr(a)[0].mT.contiguous()
    dev = "cuda"
    args = (fc3, torch.as_tensor(sc.img_ptr).to(dev), torch.as_tensor(sc.img_vec).to(dev),
            torch.as_tensor(sc.s2p).to(dev), torch.as_tensor(1.0 / np.sqrt(rng.random(n_prim) * 50 + 5)).to(dev),
            torch.as_tensor(sc.prim_frac).to(dev))
    return args, nu, e, torch.as_tensor(tetrahedra(mesh, lat)).to(dev)


@pytest.mark.parametrize("n_prim,cells,mesh,target,n_q1,spec_q1", [
    (8, (2, 2, 2), (8, 8, 8), 77, 512, 48),
    (8, (2, 2, 2), (12, 12, 12), 1001, 1728, 24),
    (31, (2, 1, 1), (4, 4, 4), 21, 64, 6),
])
def test_kernels_match_spec(n_prim, cells, mesh, target, n_q1, spec_q1):
    from chgnet_b200._lib import CudaKernels

    args, nu, e, tets = _random_case(n_prim, cells, mesh, seed=n_prim + mesh[0])
    nb = 3 * n_prim
    kern, spec = CudaKernels("cuda"), ThreePhononSpecKernels()
    q1 = torch.arange(n_q1, dtype=torch.int32, device="cuda")
    n_chunk = max(1, (1 << 28) // (56 * nb**3))  # calls of the size Phonons makes
    temps = torch.tensor([0.0, 300.0, 1000.0], dtype=torch.float64, device="cuda")
    omega = nu[target].contiguous()

    def run(k, q1s):
        p = torch.empty(len(q1s), nb, nb, nb, dtype=torch.float64, device="cuda")
        gamma = torch.zeros(3, nb, dtype=torch.float64, device="cuda")
        for s in range(0, len(q1s), n_chunk):
            ps = p[s : s + n_chunk]
            k.phonon_interaction(*args, mesh, nu, e, target, q1s[s : s + n_chunk], CUT, ps)
            k.imag_self_energy(nu, mesh, tets, target, omega, q1s[s : s + n_chunk], ps, temps, CUT, gamma)
        return p, gamma

    p, gamma = run(kern, q1)
    p2, gamma2 = run(kern, q1)
    assert torch.equal(p, p2) and torch.equal(gamma, gamma2)
    sub = q1[torch.linspace(0, n_q1 - 1, spec_q1, device="cuda").long()]
    pk, gk = run(kern, sub)
    ps, gs = run(spec, sub)
    err_p = float((pk - ps).abs().max() / ps.abs().max())
    err_g = float((gk - gs).abs().max() / gs.abs().max())
    print(f"{nb} bands, {mesh[0]}^3, target {target}: {n_q1} q1 bitwise reproducible; on {spec_q1} q1 P {err_p:.2e}, "
          f"Gamma {err_g:.2e} of max against the specification")
    assert err_p <= 1e-12 and err_g <= 1e-11


@pytest.fixture(scope="module")
def limno2_fc3():
    model = phonon_cells.model030()
    return model, model.phonons(graphgen.limno2_structure(), [2, 2, 2], third_order=True)


def test_device_fc3_against_oracle(limno2_fc3, weights030):
    model, ph = limno2_fc3
    sc, fc3, h = ph.cell, ph.force_constants3, 0.03
    n = len(sc.z)
    worst = 0.0
    for k, a, cols in ((0, 0, [0, 50, 101]), (5, 2, [7, 150])):
        hs = []
        for sgn in (1, -1):
            frac = np.array(sc.frac)
            frac[sc.p2s[k]] += sgn * h * np.linalg.inv(sc.lattice)[a]
            g = graphgen.make_crystal_graph(sc.z, frac % 1.0, sc.lattice)
            v = np.zeros((len(cols), n, 3))
            for i, c in enumerate(cols):
                v.reshape(len(cols), -1)[i, c] = 1.0
            hv = oracle_hvp(weights030, [g] * len(cols), torch.as_tensor(v.reshape(-1, 3)), None)
            hs.append(hv.reshape(len(cols), n, 3).numpy())
        want = (hs[0] - hs[1]) / (2 * h)
        for i, c in enumerate(cols):
            worst = max(worst, np.abs(fc3[k, :, c // 3, a, :, c % 3] - want[i]).max())
    scale = np.abs(fc3).max()
    asr = np.abs(fc3.sum(axis=2)).max()
    print(f"LiMnO2 2x2x2 device fc3 vs oracle central differences (h = {h}): {worst:.3e} eV/A^3 = {worst / scale:.2e} "
          f"of max|Phi3| {scale:.3e}; translational-sum residual {asr:.3e} eV/A^3 = {asr / scale:.2e} of max")
    # the fc2 agreement (4.2e-5 of max|Phi|) over 2h, relative to max|Phi3|
    fc2_scale = np.abs(ph.force_constants).max()
    assert worst <= 4.2e-5 * fc2_scale / (2 * h) * 4


def test_device_path_matches_spec_path(limno2_fc3):
    _, ph = limno2_fc3
    spec = Phonons(ph.force_constants, ph.cell, fc3=ph.force_constants3, device="cuda",
                   kernels=ThreePhononSpecKernels())
    mesh, temps = (6, 6, 6), [0.0, 300.0, 1000.0]
    q = np.array([[0.0, 0.0, 0.0], [1 / 3, 1 / 6, 0.5], [0.5, 0.5, 0.5], [-1 / 6, 2 / 3, 1 / 3]])
    got, want = ph.linewidths(mesh, q, temps), spec.linewidths(mesh, q, temps)
    err = np.abs(got["linewidths"] - want["linewidths"]).max() / np.abs(want["linewidths"]).max()
    print(f"LiMnO2 2x2x2 linewidths on 6^3 at 4 q: device vs specification path {err:.2e}")
    assert err <= 1e-9 and got["n_imaginary"] == want["n_imaginary"]
    got, want = ph.thermal_conductivity(mesh, temps), spec.thermal_conductivity(mesh, temps)
    err = np.abs(got["kappa"] - want["kappa"]).max() / np.abs(want["kappa"]).max()
    err_g = np.abs(got["linewidths"] - want["linewidths"]).max() / np.abs(want["linewidths"]).max()
    print(f"LiMnO2 2x2x2 kappa on 6^3 at 0, 300, 1000 K: device vs specification path {err:.2e} (linewidths "
          f"{err_g:.2e}); kappa(300 K) diagonal {np.diag(got['kappa'][1])} W/(m K); n_imaginary {got['n_imaginary']}, "
          f"left out for Gamma = 0 {got['n_zero_linewidth'].tolist()}")
    assert err <= 1e-9 and err_g <= 1e-9
    assert got["n_imaginary"] == want["n_imaginary"]
    assert list(got["n_zero_linewidth"]) == list(want["n_zero_linewidth"])
