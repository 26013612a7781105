"""CPU (fp64): coherent one-phonon structure factors and spectra of chgnet_b200.phonons
(Phonons.dynamic_structure_factor, Phonons.powder_spectrum), with the specifications of ``chg_structure_factors`` and
``chg_broadened_spectrum`` (tests/structure_factor_kernels.py).

* closed form: an orthorhombic spring crystal (three independent chains), whose modes are polarised along the axes,
  with and without the Debye-Waller factor;
* reduction invariance: |F| does not depend on the reciprocal-lattice vector G that reduces Q (LiMnO2 2x1x1, atoms off
  the origin), which pins the sign of the phase exp(-2 pi i G . x_k);
* completeness, sum_nu nu S+ / C = |K|^2 sum_k b_k^2 exp(-2 W_k) / m_k at T = 0, and detailed balance;
* the powder map against the direction mean of the per-Q spectra, chunking, and invalid inputs."""
import math
import os
import re

import numpy as np
import pytest
import torch

from chgnet_b200 import _lib
from chgnet_b200.phonons import (DEGENERACY_THZ, DISPLACEMENT_A2_AMU_THZ, H_OVER_KB_K_PER_THZ, THERMAL_CUTOFF_THZ,
                                 fibonacci_directions)
from phonon_cells import limno2_211_spec, springs
from structure_factor_kernels import StructureFactorSpecKernels

C = DISPLACEMENT_A2_AMU_THZ
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = (3.0, 1.7, 4.4)  # spring constants per axis (eV/A^2)
B_AL = 3.449  # a scattering length for the spring crystal's Al (fm); any value will do
# scattering lengths for LiMnO2 (fm): distinct values of both signs, so that no species drops out
B_LIMNO2 = {3: -1.90, 25: -3.73, 8: 5.80}


def _sqw_kernels(ph):
    ph.kernels = StructureFactorSpecKernels()
    return ph


@pytest.fixture(scope="module")
def spring_crystal():
    ph, nu_max = springs([3, 3, 3], ks=KS)
    return _sqw_kernels(ph), nu_max


@pytest.fixture(scope="module")
def limno2(weights030):
    return _sqw_kernels(limno2_211_spec(weights030))


def _bose(nu, t):
    return 1.0 / math.expm1(H_OVER_KB_K_PER_THZ * nu / t) if t > 0 else 0.0


def _chain_u(nu_max, n, t, m):
    """U_cc of one chain on an n-point mesh: C / (m n) sum_{j=1}^{n-1} coth(h nu_j / 2 k T) / nu_j."""
    nu = nu_max * np.sin(np.pi * np.arange(1, n) / n)
    coth = 1.0 / np.tanh(H_OVER_KB_K_PER_THZ * nu / (2 * t)) if t > 0 else np.ones_like(nu)
    return C / (m * n) * float((coth / nu).sum())


def test_header_chunk_count_matches_binding():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "chgnet_b200.h")).read(), flags=re.S)
    assert int(re.search(r"#define CHG_SQW_MAX_CHUNKS\s+(\d+)", src).group(1)) == _lib.SQW_MAX_CHUNKS


@pytest.mark.parametrize("dw_mesh", [None, (4, 5, 6)])
def test_spring_crystal_closed_form(spring_crystal, dw_mesh):
    ph, nu_max = spring_crystal
    m, a = ph.masses[0], np.diag(ph.cell.prim_lattice)
    qs = np.array([[0.3, 0.2, 0.1], [1.2, 0.4, -0.3], [0.35, 2.15, -0.45], [-1.27, 0.61, 3.08],  # off the axes
                   [0.3, 0.0, 0.0], [0.0, 1.25, 0.0], [0.0, 0.0, -2.4], [1.0, 0.0, 0.4]])  # on axes and planes
    temps = np.array([0.0, 300.0])
    out = ph.dynamic_structure_factor(qs, temps, {13: B_AL}, debye_waller_mesh=dw_mesh)
    assert out["n_imaginary"] == 0
    worst = 0.0
    for ti, t in enumerate(temps):
        u = np.zeros(3) if dw_mesh is None else np.array([_chain_u(nu_max[c], dw_mesh[c], t, m) for c in range(3)])
        for r, big_q in enumerate(qs):
            k = 2 * np.pi * big_q / a
            nu = nu_max * np.abs(np.sin(np.pi * big_q))
            w = 0.5 * float((k * k * u).sum())
            want = np.array([C * (_bose(nu[c], t) + 1.0) * B_AL**2 * math.exp(-2 * w) * k[c] ** 2 / (m * nu[c])
                             if nu[c] >= THERMAL_CUTOFF_THZ else 0.0 for c in range(3)])
            order = np.argsort(nu, kind="stable")
            assert np.all(np.diff(nu[order])[nu[order][1:] > THERMAL_CUTOFF_THZ] > 1e-3)  # no degenerate branches
            got = out["stokes"][ti, r]
            np.testing.assert_allclose(out["frequencies"][r][nu[order] >= THERMAL_CUTOFF_THZ],
                                       nu[order][nu[order] >= THERMAL_CUTOFF_THZ], rtol=1e-12)
            err = np.abs(got - want[order]).max() / np.abs(want).max()
            worst = max(worst, err)
    print(f"spring crystal closed form, Debye-Waller mesh {dw_mesh}: {worst:.2e}")
    assert worst <= 1e-12


def _set_sums(nu, s):
    """Sums of s [..., 3n] over the degenerate sets (adjacent |d nu| < DEGENERACY_THZ) of each row of nu [Q, 3n],
    placed at each set's first mode (0 elsewhere)."""
    out = np.zeros_like(s)
    for r in range(nu.shape[0]):
        start = 0
        for m in range(1, nu.shape[1] + 1):
            if m == nu.shape[1] or abs(nu[r, m] - nu[r, m - 1]) >= DEGENERACY_THZ:
                out[..., r, start] = s[..., r, start:m].sum(-1)
                start = m
    return out


def _rows(ph, q_red, g, temps, b, dw_mesh=None):
    """(nu [Q, 3n], S+ [T, Q, 3n], S- [T, Q, 3n]) through ``_structure_factor_chunks`` with the given reduction."""
    u = ph._debye_waller(dw_mesh, temps)[0]
    t = torch.as_tensor(temps).to(ph.device)
    nus, ws = [], []
    for _, nu, w, _ in ph._structure_factor_chunks(q_red, g, u, t, ph._scattering_coefficients(b)):
        nus.append(nu.cpu().numpy())
        ws.append(w.cpu().numpy())
    nu, w = np.concatenate(nus), np.concatenate(ws, axis=1)
    return nu, w[..., 0], w[..., 1]


def test_reduction_invariance(limno2):
    rng = np.random.default_rng(7)
    big_q = rng.uniform(-2.5, 2.5, size=(12, 3))
    temps = np.array([0.0, 300.0])
    g = np.floor(big_q + 0.5)
    ways = {"reduced": (big_q - g, g), "unreduced": (big_q, np.zeros_like(big_q))}
    shift = rng.integers(-3, 4, size=big_q.shape).astype(np.float64)
    ways["shifted G"] = (big_q - g - shift, g + shift)
    res = {name: _rows(limno2, q, gg, temps, B_LIMNO2, dw_mesh=(2, 2, 2)) for name, (q, gg) in ways.items()}
    nu0, sp0, sm0 = res["reduced"]
    ref = _set_sums(nu0, sp0)
    scale = np.abs(ref).max()
    assert scale > 0
    for name in ("unreduced", "shifted G"):
        nu, sp, sm = res[name]
        np.testing.assert_allclose(nu, nu0, atol=1e-9)
        err = max(np.abs(_set_sums(nu0, sp) - ref).max(), np.abs(_set_sums(nu0, sm) - _set_sums(nu0, sm0)).max())
        print(f"LiMnO2 2x1x1, {name} vs reduced, degenerate-set sums: {err / scale:.2e} of {scale:.3e}")
        assert err <= 1e-10 * scale


@pytest.mark.parametrize("dw_mesh", [None, (3, 4, 5)])
def test_completeness_spring_crystal(spring_crystal, dw_mesh):
    ph, _ = spring_crystal
    qs = np.array([[0.3, 0.2, 0.1], [1.2, 0.4, -0.3], [0.35, 2.15, -0.45], [-1.27, 0.61, 3.08]])
    temps = np.array([0.0, 300.0])
    out = ph.dynamic_structure_factor(qs, temps, {13: B_AL}, debye_waller_mesh=dw_mesh)
    assert np.all(out["frequencies"] >= THERMAL_CUTOFF_THZ)
    u = ph._debye_waller(dw_mesh, temps)[0]
    k = 2 * np.pi * qs @ np.linalg.inv(ph.cell.prim_lattice).T
    u0 = np.zeros(6) if u is None else u[0, 0].numpy()  # T = 0
    u33 = np.zeros((3, 3))
    u33[[0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1]] = u0
    u33[[0, 1, 2, 2, 2, 1], [0, 1, 2, 1, 0, 0]] = u0
    w = 0.5 * np.einsum("qa,ab,qb->q", k, u33, k)
    want = (k * k).sum(1) * B_AL**2 * np.exp(-2 * w) / ph.masses[0]
    got = (out["frequencies"] * out["stokes"][0]).sum(1) / C
    err = np.abs(got - want).max() / np.abs(want).max()
    print(f"completeness, spring crystal, Debye-Waller mesh {dw_mesh}: {err:.2e}")
    assert err <= 1e-12


def test_completeness_limno2(limno2):
    """The sum rule on the rows where LiMnO2 2x1x1 has no excluded mode."""
    rng = np.random.default_rng(3)
    qs = rng.uniform(-2.0, 2.0, size=(40, 3))
    out = limno2.dynamic_structure_factor(qs, [0.0], B_LIMNO2, debye_waller_mesh=(2, 2, 2))
    kept = np.all(out["frequencies"] >= THERMAL_CUTOFF_THZ, axis=1)
    print(f"LiMnO2 2x1x1: {int(kept.sum())} of {len(qs)} Q without an excluded mode")
    assert kept.sum() >= 5
    u = limno2._debye_waller((2, 2, 2), np.array([0.0]))[0][0].numpy()  # [n, 6]
    u33 = np.zeros((len(u), 3, 3))
    u33[:, [0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1]] = u
    u33[:, [0, 1, 2, 2, 2, 1], [0, 1, 2, 1, 0, 0]] = u
    k = 2 * np.pi * qs @ np.linalg.inv(limno2.cell.prim_lattice).T
    w = 0.5 * np.einsum("qa,kab,qb->qk", k, u33, k)
    b = np.array([B_LIMNO2[int(z)] for z in limno2.cell.prim_z])
    want = (k * k).sum(1) * (b**2 * np.exp(-2 * w) / limno2.masses).sum(1)
    got = (out["frequencies"] * out["stokes"][0]).sum(1) / C
    err = np.abs(got - want)[kept].max() / np.abs(want[kept]).max()
    print(f"completeness, LiMnO2 2x1x1: {err:.2e}")
    assert err <= 1e-12


def test_detailed_balance(limno2):
    rng = np.random.default_rng(11)
    temps = np.array([0.0, 10.0, 300.0, 1500.0])
    out = limno2.dynamic_structure_factor(rng.uniform(-1.5, 1.5, size=(10, 3)), temps, B_LIMNO2)
    nu = out["frequencies"]
    kept = nu >= THERMAL_CUTOFF_THZ
    for ti, t in enumerate(temps):
        sp, sm = out["stokes"][ti], out["anti_stokes"][ti]
        assert np.all(sp[~kept] == 0) and np.all(sm[~kept] == 0)
        want = sp * np.exp(-H_OVER_KB_K_PER_THZ * np.where(kept, nu, 1.0) / t) if t > 0 else np.zeros_like(sp)
        assert np.abs(sm - want)[kept].max() <= 1e-12 * np.abs(sp).max()


def test_gamma_modes_and_bragg_point(limno2):
    """At Q = G (q = Gamma) the three modes of smallest |nu| are returned as 0 and get S = 0."""
    out = limno2.dynamic_structure_factor([1.0, -2.0, 1.0], [300.0], B_LIMNO2)
    raw = limno2.frequencies([0.0, 0.0, 0.0])
    acoustic = np.argsort(np.abs(raw), kind="stable")[:3]
    assert np.all(out["qpoints"] == 0)
    assert np.all(out["frequencies"][acoustic] == 0) and np.all(out["stokes"][:, acoustic] == 0)
    rest = np.setdiff1d(np.arange(len(raw)), acoustic)
    np.testing.assert_allclose(out["frequencies"][rest], raw[rest], rtol=1e-12)
    assert np.all(out["stokes"][:, out["frequencies"] < THERMAL_CUTOFF_THZ] == 0)
    assert np.abs(out["stokes"]).max() > 0


def _direction_mean(ph, qm, n_dir, omega, temps, b, width, dw_mesh):
    """The mean over the Fibonacci directions of the per-Q spectra, each Q evaluated on its own."""
    i = np.arange(n_dir)
    z = 1 - (2 * i + 1) / n_dir
    phi = i * np.pi * (3 - np.sqrt(5))
    d = np.stack([np.sqrt(1 - z * z) * np.cos(phi), np.sqrt(1 - z * z) * np.sin(phi), z], 1)
    lat = ph.cell.prim_lattice
    out = np.zeros((len(temps), len(qm), len(omega)))
    for mi, q in enumerate(qm):
        for di in range(n_dir):
            big_q = (q * d[di]) @ lat.T / (2 * np.pi)
            r = ph.dynamic_structure_factor(big_q, temps, b, debye_waller_mesh=dw_mesh, frequency_points=omega,
                                            width=width)
            out[:, mi] += r["spectrum"] / n_dir
    return out


@pytest.mark.parametrize("crystal", ["springs", "limno2"])
def test_powder_is_the_direction_mean(request, crystal, spring_crystal):
    if crystal == "springs":
        ph, b, omega = spring_crystal[0], {13: B_AL}, np.linspace(-14.0, 14.0, 57)
    else:
        ph, b, omega = request.getfixturevalue("limno2"), B_LIMNO2, np.linspace(-20.0, 30.0, 51)
    qm, n_dir, temps, width = np.array([0.0, 1.3, 4.1]), 7, np.array([0.0, 300.0]), 0.8
    got = ph.powder_spectrum(qm, omega, temps, b, width=width, n_directions=n_dir, debye_waller_mesh=(2, 2, 2))
    want = _direction_mean(ph, qm, n_dir, omega, temps, b, width, (2, 2, 2))
    scale = np.abs(want).max()
    err = np.abs(got["spectrum"] - want).max() / scale
    print(f"{crystal}: powder map vs the direction mean of the per-Q spectra {err:.2e} of {scale:.3e}")
    assert err <= 1e-12
    assert np.all(got["spectrum"][:, 0] == 0)  # |Q| = 0: K = 0
    assert got["spectrum"].shape == (2, 3, len(omega))


def test_spectrum_is_the_broadened_modes(limno2):
    """spectrum = sum over modes of the two Gaussian terms, from the returned S+ and S- (a plain loop)."""
    omega, width = np.linspace(-25.0, 25.0, 101), 1.1
    sigma = width / (2 * math.sqrt(2 * math.log(2)))
    out = limno2.dynamic_structure_factor([0.31, -0.72, 1.4], [300.0], B_LIMNO2, frequency_points=omega,
                                          width=width)
    want = np.zeros_like(omega)
    for nu, sp, sm in zip(out["frequencies"], out["stokes"][0], out["anti_stokes"][0]):
        for x, s in ((omega - nu, sp), (omega + nu, sm)):
            want += s * np.where(np.abs(x) <= 8 * sigma, np.exp(-x * x / (2 * sigma**2)), 0) / (
                sigma * np.sqrt(2 * np.pi))
    assert np.abs(out["spectrum"][0] - want).max() <= 1e-13 * np.abs(want).max()
    # integrated over a fine grid, the spectrum holds sum (S+ + S-)
    fine = np.linspace(-40.0, 40.0, 16001)
    r = limno2.dynamic_structure_factor([0.31, -0.72, 1.4], [300.0], B_LIMNO2, frequency_points=fine, width=width)
    total = r["spectrum"][0].sum() * (fine[1] - fine[0])
    assert abs(total - (r["stokes"] + r["anti_stokes"]).sum()) <= 1e-9 * total


def test_chunking(limno2):
    """Tiny eigh chunks (powder groups straddle them) give the result of one chunk."""
    qm, omega, temps = np.array([0.7, 2.2, 3.3]), np.linspace(-20.0, 30.0, 41), np.array([300.0])
    whole = limno2.powder_spectrum(qm, omega, temps, B_LIMNO2, width=1.0, n_directions=5)
    big_q = np.random.default_rng(5).uniform(-2, 2, size=(7, 3))
    whole_q = limno2.dynamic_structure_factor(big_q, temps, B_LIMNO2, frequency_points=omega, width=1.0)
    batch = limno2.eigh_batch
    try:
        limno2.eigh_batch = 3
        chunked = limno2.powder_spectrum(qm, omega, temps, B_LIMNO2, width=1.0, n_directions=5)
        chunked_q = limno2.dynamic_structure_factor(big_q, temps, B_LIMNO2, frequency_points=omega, width=1.0)
    finally:
        limno2.eigh_batch = batch
    assert np.abs(chunked["spectrum"] - whole["spectrum"]).max() <= 1e-13 * np.abs(whole["spectrum"]).max()
    assert np.abs(chunked_q["spectrum"] - whole_q["spectrum"]).max() <= 1e-13 * np.abs(whole_q["spectrum"]).max()
    assert chunked["n_imaginary"] == whole["n_imaginary"]


def test_single_q_and_outputs(limno2):
    one = limno2.dynamic_structure_factor([0.2, 0.3, -0.4], [0.0, 300.0], B_LIMNO2, debye_waller_mesh=(2, 2, 2),
                                          frequency_points=np.linspace(0, 20, 11), width=0.5)
    many = limno2.dynamic_structure_factor([[0.2, 0.3, -0.4]], [0.0, 300.0], B_LIMNO2, debye_waller_mesh=(2, 2, 2),
                                           frequency_points=np.linspace(0, 20, 11), width=0.5)
    n3 = 3 * len(limno2.p2s)
    assert one["frequencies"].shape == (n3,) and one["stokes"].shape == (2, n3) and one["spectrum"].shape == (2, 11)
    assert np.array_equal(one["stokes"], many["stokes"][:, 0]) and np.array_equal(one["spectrum"], many["spectrum"][:, 0])
    td = limno2.thermal_displacement_matrices((2, 2, 2), [0.0, 300.0])
    assert one["debye_waller_n_imaginary"] == td["n_imaginary"]
    freqs = limno2.frequencies([0.2, 0.3, -0.4])
    assert one["n_imaginary"] == int((freqs < -THERMAL_CUTOFF_THZ).sum())


def test_fibonacci_directions():
    d = fibonacci_directions(500)
    np.testing.assert_allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-15)
    assert np.abs(d.mean(0)).max() < 1e-2  # evenly spread


def test_invalid_inputs(limno2):
    ph, b = limno2, B_LIMNO2
    with pytest.raises(ValueError, match="finite"):
        ph.dynamic_structure_factor([0.1, np.nan, 0.0], [300.0], b)
    with pytest.raises(ValueError, match="temperatures"):
        ph.dynamic_structure_factor([0.1, 0.2, 0.0], [-1.0], b)
    with pytest.raises(ValueError, match="temperatures"):
        ph.powder_spectrum([1.0], [1.0], [np.inf], b, width=1.0)
    with pytest.raises(ValueError, match="width"):
        ph.dynamic_structure_factor([0.1, 0.2, 0.0], [300.0], b, frequency_points=[1.0], width=0.0)
    with pytest.raises(ValueError, match="width"):
        ph.dynamic_structure_factor([0.1, 0.2, 0.0], [300.0], b, frequency_points=[1.0])
    with pytest.raises(ValueError, match="width"):
        ph.powder_spectrum([1.0], [1.0], [300.0], b, width=-1.0)
    with pytest.raises(ValueError, match="n_directions"):
        ph.powder_spectrum([1.0], [1.0], [300.0], b, width=1.0, n_directions=0)
    with pytest.raises(ValueError, match="q_magnitudes"):
        ph.powder_spectrum([-1.0], [1.0], [300.0], b, width=1.0)
    with pytest.raises(ValueError, match="q_magnitudes"):
        ph.powder_spectrum([np.nan], [1.0], [300.0], b, width=1.0)
    with pytest.raises(ValueError, match="atomic number 25"):
        ph.dynamic_structure_factor([0.1, 0.2, 0.0], [300.0], {3: -1.9, 8: 5.8})
    with pytest.raises(ValueError, match="atomic number 8"):
        ph.powder_spectrum([1.0], [1.0], [300.0], {3: -1.9, 25: -3.73, 8: float("nan")}, width=1.0)


def test_broadening_calls_split_by_the_scratch_budget(limno2):
    """With a scratch budget of a few groups, the broadening runs in several calls per eigh chunk (groups split
    between them) and gives the result of one call."""
    from chgnet_b200._lib import sqw_scratch_doubles

    qm, omega, temps = np.array([0.7, 2.2, 3.3]), np.linspace(-20.0, 30.0, 41), np.array([0.0, 300.0])
    big_q = np.random.default_rng(6).uniform(-2, 2, size=(9, 3))
    whole = limno2.powder_spectrum(qm, omega, temps, B_LIMNO2, width=1.0, n_directions=5)
    whole_q = limno2.dynamic_structure_factor(big_q, temps, B_LIMNO2, frequency_points=omega, width=1.0)
    budget = limno2.sqw_chunk_bytes
    calls = []
    broadened = limno2.kernels.broadened_spectrum

    def counted(nu, *args):
        calls.append(nu.shape[0])
        broadened(nu, *args)

    try:
        limno2.kernels.broadened_spectrum = counted
        limno2.sqw_chunk_bytes = 8 * sqw_scratch_doubles(5, 3 * len(limno2.p2s), 2, 0, 5, 41)  # one group
        split = limno2.powder_spectrum(qm, omega, temps, B_LIMNO2, width=1.0, n_directions=5)
        limno2.sqw_chunk_bytes = 8 * 3 * 2 * 41  # three one-row groups
        split_q = limno2.dynamic_structure_factor(big_q, temps, B_LIMNO2, frequency_points=omega, width=1.0)
    finally:
        limno2.sqw_chunk_bytes = budget
        del limno2.kernels.broadened_spectrum
    assert max(calls) < 5 and len(calls) > 4
    assert np.abs(split["spectrum"] - whole["spectrum"]).max() <= 1e-13 * np.abs(whole["spectrum"]).max()
    assert np.abs(split_q["spectrum"] - whole_q["spectrum"]).max() <= 1e-13 * np.abs(whole_q["spectrum"]).max()


def test_scratch_size():
    from chgnet_b200._lib import SQW_MAX_CHUNKS, sqw_scratch_doubles

    assert sqw_scratch_doubles(4096, 24, 31, 0, 1, 401) == 4096 * 31 * 401  # one chunk of one-row groups
    assert sqw_scratch_doubles(4096, 24, 1, 0, 1000, 401) == SQW_MAX_CHUNKS * 5 * 401  # 5 groups, 750 tiles of 32
    assert sqw_scratch_doubles(10, 3, 2, 995, 1000, 7) == 1 * 2 * 2 * 7  # 10 rows x 3 modes: one tile, two groups
    assert sqw_scratch_doubles(0, 24, 1, 0, 1, 401) == 0
