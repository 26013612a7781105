"""-m gpu: coherent one-phonon structure factors and spectra on the device (Phonons.dynamic_structure_factor,
Phonons.powder_spectrum).

* ``chg_structure_factors`` against its fp64 specification (tests/structure_factor_kernels.py) at production sizes,
  random unitary eigenvectors with negative, sub-cutoff and exactly-cutoff frequencies: 8 atoms x 4 096 Q x 31
  temperatures (with and without U), 31 atoms x 1 024 Q x one temperature, one atom x 5 000 Q;
* ``chg_broadened_spectrum`` against its specification with group sizes 1 and 500 and a group straddling two calls,
  401 frequency points; both kernels bitwise reproducible, and the broadening exactly doubles on a second call;
* the device force constants of LiMnO2 2x2x2: device path against specification path (Q-points over two eigh chunks,
  a 50-shell x 200-direction powder map, Debye-Waller on 12^3), reduction invariance and completeness."""
import math

import numpy as np
import phonon_cells
import pytest
import torch

from chgnet_b200.phonons import DEGENERACY_THZ, DISPLACEMENT_A2_AMU_THZ, THERMAL_CUTOFF_THZ
from structure_factor_kernels import StructureFactorSpecKernels
from test_structure_factor_spec import B_LIMNO2, _rows, _set_sums
from test_thermal_displacements_gpu import _random_modes

pytestmark = pytest.mark.gpu

TEMPS = np.linspace(0.0, 1500.0, 31)


def _sqw_inputs(n_q, n_prim, n_t, seed, with_u=True):
    g = torch.Generator(device="cuda").manual_seed(seed + 17)
    dev, f64 = "cuda", torch.float64
    nu, e = _random_modes(n_q, n_prim, seed)
    kcart = torch.randn(n_q, 3, generator=g, device=dev, dtype=f64) * 3.0
    gvec = torch.randint(-4, 5, (n_q, 3), generator=g, device=dev).to(f64)
    frac = torch.rand(n_prim, 3, generator=g, device=dev, dtype=f64)
    coef = torch.randn(n_prim, generator=g, device=dev, dtype=f64)
    u = None
    if with_u:
        a = torch.randn(n_t, n_prim, 3, 3, generator=g, device=dev, dtype=f64) * 0.05
        u33 = a @ a.mT + 0.005 * torch.eye(3, device=dev, dtype=f64)
        u = u33[..., [0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1]].contiguous()
    temps = TEMPS[:n_t] if n_t == 31 else np.array([300.0])
    return nu, e, kcart, gvec, frac, coef, u, torch.as_tensor(temps).cuda()


@pytest.mark.parametrize("case", ["8atoms_4096q_31T", "8atoms_4096q_31T_noU", "31atoms_1024q_1T", "1atom_5000q_31T"])
def test_structure_factors_kernel_matches_spec(case):
    from chgnet_b200._lib import CudaKernels

    n_prim, n_q, n_t = {"8atoms_4096q_31T": (8, 4096, 31), "8atoms_4096q_31T_noU": (8, 4096, 31),
                        "31atoms_1024q_1T": (31, 1024, 1), "1atom_5000q_31T": (1, 5000, 31)}[case]
    args = _sqw_inputs(n_q, n_prim, n_t, seed=n_prim * 1000 + n_t, with_u=not case.endswith("noU"))
    kern = CudaKernels("cuda")

    def run(k):
        out = torch.empty(n_t, n_q, 3 * n_prim, 2, dtype=torch.float64, device="cuda")
        k.structure_factors(*args, THERMAL_CUTOFF_THZ, out)
        return out

    got, want, again = run(kern), run(StructureFactorSpecKernels()), run(kern)
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    print(f"{case}: max|kernel - spec| / max = {err:.2e} (max {scale:.3e})")
    assert err <= 1e-12
    assert torch.equal(got, again)
    nu = args[0]
    assert bool((got[:, nu < THERMAL_CUTOFF_THZ] == 0).all())


@pytest.mark.parametrize("case", ["group1", "group500", "straddle"])
def test_broadened_spectrum_kernel_matches_spec(case):
    from chgnet_b200._lib import CudaKernels

    n_prim, n_t = 8, 3
    n_q, gs = {"group1": (2048, 1), "group500": (3000, 500), "straddle": (1500, 500)}[case]
    nu, e, kcart, gvec, frac, coef, u, _ = _sqw_inputs(n_q, n_prim, 31, seed=4242 + n_q)
    t = torch.as_tensor([0.0, 300.0, 1200.0]).cuda()
    w = torch.empty(n_t, n_q, 3 * n_prim, 2, dtype=torch.float64, device="cuda")
    StructureFactorSpecKernels().structure_factors(nu, e, kcart, gvec, frac, coef, u[:n_t].contiguous(), t,
                                                   THERMAL_CUTOFF_THZ, w)
    omega = torch.linspace(-25.0, 25.0, 401, dtype=torch.float64, device="cuda")
    sigma = 0.4
    n_groups = -(-n_q // gs)
    # the straddling case: rows [0, 700) and [700, 1500) in two calls, group 1 in both
    cuts = [0, 700, n_q] if case == "straddle" else [0, n_q]
    kern = CudaKernels("cuda")

    def run(k, out=None):
        out = torch.zeros(n_t, n_groups, 401, dtype=torch.float64, device="cuda") if out is None else out
        for a, b in zip(cuts[:-1], cuts[1:]):
            k.broadened_spectrum(nu[a:b], w[:, a:b].contiguous(), a, gs, omega, sigma, out)
        return out

    got, want, again = run(kern), run(StructureFactorSpecKernels()), run(kern)
    scale = float(want.abs().max())
    err = float((got - want).abs().max()) / scale
    print(f"{case}: {n_q} rows, groups of {gs}, 401 points: max|kernel - spec| / max = {err:.2e} (max {scale:.3e})")
    assert err <= 1e-12
    assert torch.equal(got, again)
    # a second call on the same out adds exactly what the first did (one call: a straddling group's two calls
    # round in their own order)
    once = torch.zeros(n_t, n_groups, 401, dtype=torch.float64, device="cuda")
    kern.broadened_spectrum(nu[: cuts[1]], w[:, : cuts[1]].contiguous(), 0, gs, omega, sigma, once)
    twice = once.clone()
    kern.broadened_spectrum(nu[: cuts[1]], w[:, : cuts[1]].contiguous(), 0, gs, omega, sigma, twice)
    assert torch.equal(twice, 2 * once)


@pytest.fixture(scope="module")
def limno2_222():
    ph = phonon_cells.limno2_222(phonon_cells.model030())
    spec = phonon_cells.spec_phonons(ph.force_constants, ph.cell)
    spec.kernels = StructureFactorSpecKernels()
    return ph, spec


def test_device_path_matches_spec_path(limno2_222):
    ph, spec = limno2_222
    rng = np.random.default_rng(2)
    big_q = rng.uniform(-3.0, 3.0, size=(5000, 3))  # two eigh chunks of at most 4 096
    assert len(big_q) > ph.eigh_batch
    temps = np.array([0.0, 300.0])
    omega = np.linspace(-30.0, 30.0, 241)
    kw = dict(debye_waller_mesh=(12, 12, 12), frequency_points=omega, width=0.5)
    got = ph.dynamic_structure_factor(big_q, temps, B_LIMNO2, **kw)
    again = ph.dynamic_structure_factor(big_q, temps, B_LIMNO2, **kw)
    want = spec.dynamic_structure_factor(big_q, temps, B_LIMNO2, **kw)
    nu = got["frequencies"]
    np.testing.assert_allclose(nu, want["frequencies"], atol=1e-9 * np.abs(nu).max())
    errs = {}
    for key in ("stokes", "anti_stokes"):
        ref = _set_sums(nu, want[key])
        errs[key] = np.abs(_set_sums(nu, got[key]) - ref).max() / np.abs(ref).max()
    errs["spectrum"] = np.abs(got["spectrum"] - want["spectrum"]).max() / np.abs(want["spectrum"]).max()
    print(f"LiMnO2 2x2x2 device force constants, 5 000 Q, Debye-Waller 12^3: device vs specification path {errs}; "
          f"n_imaginary {got['n_imaginary']}, Debye-Waller mesh {got['debye_waller_n_imaginary']}")
    assert max(errs.values()) <= 1e-9
    assert got["n_imaginary"] == want["n_imaginary"]
    assert got["debye_waller_n_imaginary"] == want["debye_waller_n_imaginary"]
    assert np.array_equal(got["spectrum"], again["spectrum"]) and np.array_equal(got["stokes"], again["stokes"])

    qm = np.linspace(0.2, 8.0, 50)
    pw = dict(width=0.5, n_directions=200, debye_waller_mesh=(12, 12, 12))
    got_p = ph.powder_spectrum(qm, omega, [300.0], B_LIMNO2, **pw)
    want_p = spec.powder_spectrum(qm, omega, [300.0], B_LIMNO2, **pw)
    err = np.abs(got_p["spectrum"] - want_p["spectrum"]).max() / np.abs(want_p["spectrum"]).max()
    print(f"powder map 50 shells x 200 directions (10 000 Q, three eigh chunks): device vs specification {err:.2e}; "
          f"n_imaginary {got_p['n_imaginary']}")
    assert err <= 1e-9
    assert got_p["n_imaginary"] == want_p["n_imaginary"]


def test_device_reduction_invariance_and_completeness(limno2_222):
    ph, _ = limno2_222
    rng = np.random.default_rng(9)
    big_q = rng.uniform(-2.5, 2.5, size=(300, 3))
    temps = np.array([0.0, 300.0])
    g = np.floor(big_q + 0.5)
    shift = rng.integers(-3, 4, size=big_q.shape).astype(np.float64)
    nu0, sp0, _ = _rows(ph, big_q - g, g, temps, B_LIMNO2, dw_mesh=(6, 6, 6))
    ref = _set_sums(nu0, sp0)
    for name, (q, gg) in {"unreduced": (big_q, 0 * big_q), "shifted G": (big_q - g - shift, g + shift)}.items():
        nu, sp, _ = _rows(ph, q, gg, temps, B_LIMNO2, dw_mesh=(6, 6, 6))
        err = np.abs(_set_sums(nu0, sp) - ref).max() / np.abs(ref).max()
        print(f"device, {name} vs reduced: {err:.2e}")
        assert err <= 1e-10

    kept = np.all(nu0 >= THERMAL_CUTOFF_THZ, axis=1)
    assert kept.sum() >= 10
    u = ph._debye_waller((6, 6, 6), temps)[0][0].cpu().numpy()
    u33 = np.zeros((len(u), 3, 3))
    u33[:, [0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1]] = u
    u33[:, [0, 1, 2, 2, 2, 1], [0, 1, 2, 1, 0, 0]] = u
    k = 2 * math.pi * big_q @ np.linalg.inv(ph.cell.prim_lattice).T
    w = 0.5 * np.einsum("qa,kab,qb->qk", k, u33, k)
    b = np.array([B_LIMNO2[int(z)] for z in ph.cell.prim_z])
    want = (k * k).sum(1) * (b**2 * np.exp(-2 * w) / ph.masses).sum(1)
    got = (nu0 * sp0[0]).sum(1) / DISPLACEMENT_A2_AMU_THZ
    err = np.abs(got - want)[kept].max() / np.abs(want[kept]).max()
    print(f"device completeness on {int(kept.sum())} of {len(big_q)} Q: {err:.2e}; degeneracy {DEGENERACY_THZ}")
    assert err <= 1e-12


def test_spectrum_at_many_q_and_temperatures(limno2_222):
    """5 000 Q (two eigh chunks) x 31 temperatures with a spectrum: 4 096 one-row groups x 31 temperatures in one
    broadening call, against the specification path; the same with the calls split by a small scratch budget."""
    from chgnet_b200._lib import sqw_scratch_doubles

    ph, spec = limno2_222
    big_q = np.random.default_rng(4).uniform(-3.0, 3.0, size=(5000, 3))
    omega = np.linspace(-30.0, 30.0, 201)
    kw = dict(debye_waller_mesh=(8, 8, 8), frequency_points=omega, width=0.5)
    got = ph.dynamic_structure_factor(big_q, TEMPS, B_LIMNO2, **kw)
    want = spec.dynamic_structure_factor(big_q, TEMPS, B_LIMNO2, **kw)
    err = np.abs(got["spectrum"] - want["spectrum"]).max() / np.abs(want["spectrum"]).max()
    scratch = 8 * sqw_scratch_doubles(ph.eigh_batch, 24, len(TEMPS), 0, 1, len(omega))
    print(f"5 000 Q x 31 T x 201 points: device vs specification path {err:.2e}; broadening scratch of one "
          f"{ph.eigh_batch}-row call {scratch / 2**20:.0f} MiB")
    assert err <= 1e-9
    assert scratch <= ph.sqw_chunk_bytes
    budget = ph.sqw_chunk_bytes
    try:
        ph.sqw_chunk_bytes = 1 << 22  # 4 MiB: 83 rows per call here
        split = ph.dynamic_structure_factor(big_q, TEMPS, B_LIMNO2, **kw)
        powder_split = ph.powder_spectrum([1.0, 3.0, 5.0], omega, TEMPS, B_LIMNO2, width=0.5, n_directions=2000)
    finally:
        ph.sqw_chunk_bytes = budget
    # one-row groups add the same terms in the same order however the rows are split
    assert np.array_equal(split["spectrum"], got["spectrum"])
    powder = ph.powder_spectrum([1.0, 3.0, 5.0], omega, TEMPS, B_LIMNO2, width=0.5, n_directions=2000)
    err_p = np.abs(powder_split["spectrum"] - powder["spectrum"]).max() / np.abs(powder["spectrum"]).max()
    print(f"powder 3 shells x 2 000 directions x 31 T, split calls vs default: {err_p:.2e}")
    assert err_p <= 1e-13
