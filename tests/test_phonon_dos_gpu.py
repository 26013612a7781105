"""-m gpu: phonon group velocities and densities of states on the device (Phonons.group_velocities, Phonons.dos).

* ``chg_dynamical_matrix_derivatives`` against its fp64 specification (oracle/phonons.py) with synthetic force
  constants at the sizes of test_phonons_gpu.py: LiMnO2 4x4x4 on a 16^3 mesh, a 31-atom random cell 3x3x3, a
  non-diagonal supercell; bitwise reproducible and written Hermitian;
* ``chg_tetrahedron_dos`` with projections on a 24^3 mesh against its specification, with tied vertex values and
  frequency points on vertices; bitwise reproducible;
* the device force constants of LiMnO2 2x2x2: ``group_velocities`` and ``dos`` against the specification path on the
  same force constants, and the acoustic velocities near Gamma."""
import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import gamma_mesh, make_supercell, tetrahedra
from oracle.phonons import PhononSpecKernels

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", ["limno2_444_mesh16", "random31_333", "limno2_nondiagonal"])
def test_derivative_kernel_matches_spec(case):
    from chgnet_b200._lib import CudaKernels

    rng = np.random.default_rng(23)
    if case == "limno2_444_mesh16":
        sc = make_supercell(*graphgen.limno2_structure(), [4, 4, 4])
        q = gamma_mesh((16, 16, 16))
    elif case == "random31_333":
        sc = make_supercell(*graphgen.random_structure(31, 9731), [3, 3, 3])
        q = rng.uniform(-1.0, 1.0, size=(300, 3))
    else:
        sc = make_supercell(*graphgen.limno2_structure(), [[1, 1, 0], [-1, 1, 0], [0, 0, 2]])
        q = rng.uniform(-0.5, 0.5, size=(1000, 3))
    n_prim, n = len(sc.p2s), len(sc.s2p)
    fc = rng.normal(size=(n_prim, n, 3, 3))
    dev = torch.device("cuda")
    args = [torch.as_tensor(x).to(dev) for x in (fc, sc.img_ptr, sc.img_vec, sc.s2p,
                                                   rng.uniform(0.1, 0.6, size=n_prim), q, sc.prim_lattice)]
    n3 = 3 * n_prim
    kern = CudaKernels(dev)
    got = torch.full((len(q), 3, n3, n3), float("nan"), dtype=torch.complex128, device=dev)
    kern.dynamical_matrix_derivatives(*args, got)
    again = torch.empty_like(got)
    kern.dynamical_matrix_derivatives(*args, again)
    want = torch.empty_like(got)
    PhononSpecKernels().dynamical_matrix_derivatives(*args, want)
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    print(case, f"max|dD/dQ - spec| / max|dD/dQ| = {err:.2e} (max {scale:.3e})")
    assert err <= 1e-10
    assert torch.equal(torch.view_as_real(got), torch.view_as_real(again))
    assert torch.equal(got, got.conj().transpose(-1, -2))


def test_tetrahedron_dos_kernel_matches_spec():
    from chgnet_b200._lib import CudaKernels

    rng = np.random.default_rng(29)
    mesh = (24, 24, 24)
    n_q, n_band, n_proj = 24**3, 24, 7  # 7 projections: one full and one partial group of the kernel
    # values on a 1/8 THz grid: vertices tie often, and every frequency point below sits on possible vertex values
    freqs = np.sort(np.round(rng.uniform(-2.0, 20.0, size=(n_q, n_band)) * 8) / 8, axis=1)
    proj = rng.uniform(0.0, 1.0, size=(n_q, n_band, n_proj))
    omega = np.arange(-2.5, 20.5, 0.125)
    lat = graphgen.limno2_structure()[2]
    dev = torch.device("cuda")
    f, p, w = (torch.as_tensor(x).to(dev) for x in (freqs, proj, omega))
    tets = torch.as_tensor(tetrahedra(mesh, lat)).to(dev)
    kern = CudaKernels(dev)

    def run(k, with_proj=True):
        out = [torch.full((len(omega),), float("nan"), dtype=torch.float64, device=dev) for _ in range(2)]
        pd = torch.full((n_proj, len(omega)), float("nan"), dtype=torch.float64, device=dev) if with_proj else None
        k.tetrahedron_dos(f, mesh, tets, w, out[0], out[1], p if with_proj else None, pd)
        return out + ([pd] if with_proj else [])

    got, again, want = run(kern), run(kern), run(PhononSpecKernels())
    plain = run(kern, with_proj=False)
    for name, a, b, c in zip(("dos", "idos", "pdos"), got, again, want):
        scale = float(c.abs().max())
        err = float((a - c).abs().max()) / scale
        print(f"tetrahedron dos 24^3, {n_band} bands, {len(omega)} points: {name} max|kernel - spec| / max = {err:.2e}")
        assert err <= 1e-10 and torch.equal(a, b)
    assert torch.equal(plain[0], got[0]) and torch.equal(plain[1], got[1])
    assert abs(float(got[1][-1]) - n_band) <= 1e-12 * n_band


@pytest.fixture(scope="module")
def limno2_222():
    ph = phonon_cells.limno2_222(phonon_cells.model030())
    return ph, phonon_cells.spec_phonons(ph.force_constants, ph.cell)


def test_group_velocities_and_dos_match_spec_path(limno2_222):
    ph, spec = limno2_222
    rng = np.random.default_rng(31)
    q = rng.uniform(-0.5, 0.5, size=(500, 3))
    v, vs = ph.group_velocities(q), spec.group_velocities(q)
    # modes closer than 1e-2 THz are compared by their sum: a velocity of one mode of a near-degenerate pair is
    # ill-conditioned (its eigenvector turns by rounding / gap), the pair's sum is not
    nu = spec.frequencies(q)
    cluster = np.concatenate([np.zeros((len(q), 1), int), np.cumsum(np.diff(nu, axis=1) > 1e-2, axis=1)], axis=1)
    sums = np.zeros((2, len(q), 24, 3))
    for i, x in enumerate((v, vs)):
        np.add.at(sums[i], (np.arange(len(q))[:, None], cluster), x)
    err_v = np.abs(sums[0] - sums[1]).max() / np.abs(vs).max()
    mesh = (10, 10, 10)
    d, ds = ph.dos(mesh, projected=True), spec.dos(mesh, projected=True)
    print(f"LiMnO2 2x2x2 device force constants: group velocities vs spec path {err_v:.2e} of max|v| "
          f"({np.abs(vs).max():.1f} THz A)")
    assert v.shape == (500, 24, 3) and err_v <= 1e-9
    assert np.abs(d["frequency_points"] - ds["frequency_points"]).max() <= 1e-9 * np.abs(ds["frequency_points"]).max()
    for k in ("total_dos", "integrated_dos", "projected_dos"):
        err = np.abs(d[k] - ds[k]).max() / np.abs(ds[k]).max()
        print(f"  dos {mesh}: {k} vs spec path {err:.2e}")
        assert err <= 1e-9, k
    assert abs(d["integrated_dos"][-1] - 24) <= 1e-12
    assert np.abs(d["projected_dos"].sum(0) - d["total_dos"]).max() <= 1e-12 * d["total_dos"].max()


def test_acoustic_velocities_near_gamma(limno2_222):
    ph, _ = limno2_222
    lat = ph.cell.prim_lattice
    speeds = {}
    for step in (1e-3, 2e-3):
        q = step * np.eye(3) @ lat.T  # Q = step along x, y, z (1/A)
        nu, v = ph.frequencies(q), ph.group_velocities(q)
        acoustic = np.argsort(np.abs(nu), axis=1)[:, :3]
        s = np.linalg.norm(np.take_along_axis(v, acoustic[:, :, None], axis=1), axis=2)
        speeds[step] = np.sort(s, axis=1)
    print("acoustic |v| (THz A = 100 m/s) along x, y, z at |Q| = 1e-3 and 2e-3 1/A:\n", speeds[1e-3], "\n", speeds[2e-3])
    assert np.isfinite(speeds[1e-3]).all() and (speeds[1e-3] > 1.0).all()
    assert np.abs(speeds[1e-3] - speeds[2e-3]).max() <= 1e-2 * speeds[1e-3].max()
