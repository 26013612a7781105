"""CPU (fp64): frequency-resolved three-phonon self-energies and phonon spectral functions of chgnet_b200.phonons
(Phonons.spectral_function) with the specification of ``chg_self_energy_spectrum`` (tests/spectral_function_kernels.py).

* at the target's own band frequencies the spectrum is ``imag_self_energy`` (the diagonal band = point);
* with P = 1/N it is 18 pi / h^2 (N2(1) + N2(2)) of ``joint_dos`` on the whole grid, which the flipped class-1 sign
  fails at T > 0;
* the closed-form real part against a principal-value quadrature of the interpolated Gamma, at w = 0, on and off the
  grid and beyond it; Delta even (the transform of an odd Gamma);
* the first-moment sum rule of A, which a flipped Delta and a Delta without the odd extension fail;
* the weak-coupling limit: Gamma and Delta scale as s^2 with fc3 s, and A tends to a Lorentzian;
* chunking, independent temperatures, input errors and the header's chunk limit."""
import math
import os
import re

import numpy as np
import pytest
import torch
from scipy import integrate

from chgnet_b200.phonons import (H_EV_PER_THZ, THERMAL_CUTOFF_THZ, Phonons, _hat_matrix, _hilbert_matrix)
from phonon_cells import limno2_211, springs
from spectral_function_kernels import SpectralFunctionSpecKernels
from test_three_phonon_spec import KS, _chain_fc3, _random_symmetric_fc3

CUT = THERMAL_CUTOFF_THZ
f64 = torch.float64
K = 18 * math.pi / H_EV_PER_THZ**2
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spec(fc, sc, fc3, **kw):
    return Phonons(fc, sc, fc3=fc3, device="cpu", kernels=SpectralFunctionSpecKernels(**kw))


@pytest.fixture(scope="module")
def limno2(weights030):
    sc, _, fc = limno2_211(weights030)
    return sc, fc, _random_symmetric_fc3(sc, 3)[1]


def _springs():
    ph0, _ = springs((3, 3, 3), ks=KS)
    return _spec(ph0.force_constants, ph0.cell, _chain_fc3(ph0.cell)), (3, 3, 3)


@pytest.mark.parametrize("cell", ["springs_333", "limno2_211"])
def test_band_frequencies_give_imag_self_energy(cell, request):
    if cell == "springs_333":
        ph, mesh = _springs()
        targets = (1, 5, 13, 26)
    else:
        sc, fc, fc3 = request.getfixturevalue("limno2")
        ph, mesh = _spec(fc, sc, fc3), (2, 2, 2)
        targets = (0, 3, 6)
    mesh_t, nu, e, _, tets, _ = ph._three_phonon_mesh(mesh, None)
    n_mesh, nb = nu.shape
    t = torch.tensor([0.0, 300.0, 1000.0], dtype=f64)
    q1 = torch.arange(n_mesh, dtype=torch.int32)
    worst = 0.0
    for target in targets:
        p = ph._interactions(mesh_t, nu, e, target, q1)
        omega = nu[target].contiguous()
        want = torch.zeros(3, nb, dtype=f64)
        got = torch.zeros(3, nb, nb, dtype=f64)
        ph.kernels.imag_self_energy(nu, mesh_t, tets, target, omega, q1, p, t, CUT, want)
        ph.kernels.self_energy_spectrum(nu, mesh_t, tets, target, omega, q1, p, t, CUT, got)
        worst = max(worst, float((got.diagonal(dim1=1, dim2=2) - want).abs().max() / want.abs().max()))
    print(f"{cell}: self_energy_spectrum at the band frequencies vs imag_self_energy {worst:.2e}")
    assert worst <= 1e-13


def _jdos_link(ph, mesh, temps):
    """max over the targets of |Gamma(w_k) - K (N2(1) + N2(2))(w_k)| / max, P = 1/N, on 201 points to 2 nu_max: at
    every point but w_0 = 0, where Gamma is 0 (below the cutoff) and joint_dos' doubled class-1 term is not."""
    mesh_t, nu, _, _, tets, _ = ph._three_phonon_mesh(mesh, None)
    n_mesh, nb = nu.shape
    grid = torch.arange(201, dtype=f64) * (float(2 * nu.max()) / 200)
    t = torch.as_tensor(np.array(temps))
    q1 = torch.arange(n_mesh, dtype=torch.int32)
    p = torch.full((n_mesh, nb, nb, nb), 1.0 / n_mesh, dtype=f64)
    coords = np.stack(np.unravel_index(np.arange(n_mesh), mesh), 1) / np.array(mesh)
    jd = ph.joint_dos(mesh, coords, grid.numpy(), temps)["weighted_jdos"]  # [T, N, 2, F]
    worst = 0.0
    for target in range(n_mesh):
        gamma = torch.zeros(len(temps), nb, len(grid), dtype=f64)
        ph.kernels.self_energy_spectrum(nu, mesh_t, tets, target, grid, q1, p, t, CUT, gamma)
        want = K * jd[:, target].sum(1)  # [T, F], the same for every band
        assert np.all(gamma[:, :, 0].numpy() == 0)
        worst = max(worst, np.abs(gamma[:, :, 1:].numpy() - want[:, None, 1:]).max() / np.abs(want).max())
    return worst


def test_constant_p_gives_joint_dos(limno2):
    sc, fc, _ = limno2
    zero = np.zeros((len(sc.p2s), len(sc.z), len(sc.z), 3, 3, 3))
    mesh = (3, 2, 2)
    err = _jdos_link(_spec(fc, sc, zero), mesh, [0.0, 300.0, 1000.0])
    bad0 = _jdos_link(_spec(fc, sc, zero, class1_sign=-1.0), mesh, [0.0])
    bad = _jdos_link(_spec(fc, sc, zero, class1_sign=-1.0), mesh, [300.0])
    print(f"LiMnO2 2x1x1 on 3x2x2, P = 1/N: Gamma(w) vs 18 pi / h^2 (N2(1) + N2(2)) {err:.2e}; with the class-1 "
          f"sign flipped {bad0:.2e} at 0 K, {bad:.2e} at 300 K")
    assert err <= 1e-13 and bad0 <= 1e-13 and bad > 1e-3


def _pv_delta(gamma_k, h, w):
    """(1/pi) PV int_0^inf G(x) [1 / (w - x) - 1 / (w + x)] dx for the piecewise-linear G of the grid values gamma_k
    (0 beyond the last hat), by quadrature: QUADPACK's Cauchy-weight rule on the interval that holds w inside, the
    symmetric form int_0^h (G(w + u) - G(w - u)) / u du around a grid point w, plain quadrature elsewhere."""
    m = len(gamma_k)
    xs = np.arange(m + 1) * h
    vals = np.append(gamma_k, 0.0)

    def g(x):
        return np.interp(x, xs, vals, left=0.0, right=0.0)

    total = 0.0
    j = int(round(w / h))
    on_grid = abs(w - j * h) <= 1e-12 * h and 0 < j < m + 1
    for k in range(m):
        a, b = xs[k], xs[k + 1]
        if on_grid and k in (j - 1, j):
            continue
        if a < w < b:
            total -= integrate.quad(g, a, b, weight="cauchy", wvar=w, epsabs=1e-14, epsrel=1e-12)[0]
        else:
            total += integrate.quad(lambda x: g(x) / (w - x), a, b, epsabs=1e-14, epsrel=1e-12)[0]
        total -= integrate.quad(lambda x: g(x) / (w + x), a, b, epsabs=1e-14, epsrel=1e-12)[0]
    if on_grid:
        total -= integrate.quad(lambda u: (g(w + u) - g(w - u)) / u, 0, h, epsabs=1e-14, epsrel=1e-12)[0]
        for k in (j - 1, j):
            if k < m:
                total -= integrate.quad(lambda x: g(x) / (w + x), xs[k], xs[k + 1], epsabs=1e-14, epsrel=1e-12)[0]
    return total / math.pi


def test_real_part_is_the_hilbert_transform():
    rng = np.random.default_rng(4)
    m, h = 41, 0.25
    gamma = rng.random(m) * np.sin(np.linspace(0, math.pi, m)) ** 2  # 0 at both ends
    gamma[0] = 0.0
    gamma[-2] += 0.3  # a sizeable value next to the last point
    grid = torch.arange(m, dtype=f64) * h
    pts = np.array([0.0, h, 7 * h, (m - 1) * h, 0.3 * h, 13.37 * h, (m - 1.5) * h, (m - 0.5) * h, (m + 3.2) * h,
                    3 * m * h])
    got = (_hilbert_matrix(torch.as_tensor(pts), grid, h) @ torch.as_tensor(gamma)).numpy()
    want = np.array([_pv_delta(gamma, h, w) for w in pts])
    err = np.abs(got - want).max() / np.abs(want).max()
    neg = (_hilbert_matrix(torch.as_tensor(-pts), grid, h) @ torch.as_tensor(gamma)).numpy()
    print(f"closed-form Delta vs principal-value quadrature at {len(pts)} points {err:.2e}; Delta(0) = {got[0]:.4f} "
          f"= -(2 / pi) int Gamma / w")
    assert err <= 1e-12
    assert got[0] < 0 and np.array_equal(neg, got)
    # the interpolant: the grid values at the grid points, linear between them, 0 beyond the last hat
    hat = _hat_matrix(torch.as_tensor(pts), grid, h) @ torch.as_tensor(gamma)
    want_hat = np.interp(pts, np.arange(m + 1) * h, np.append(gamma, 0.0), right=0.0)
    assert np.abs(hat.numpy() - want_hat).max() <= 1e-15


def _a_from(gamma, nu, omega, grid, h, hilbert):
    """A [..., F] from gamma [..., M] and nu [...] with the real part of the matrix function ``hilbert``."""
    w = torch.as_tensor(omega)
    g = gamma @ _hat_matrix(w, grid, h).T
    d = gamma @ hilbert(w, grid, h).T
    v = nu[..., None]
    den = (w * w - v * v - 2 * v * d) ** 2 + 4 * v * v * g * g
    return torch.where(g != 0, 4 * v * v * g / (math.pi * torch.where(g != 0, den, 1.0)), 0.0), g, d


def _no_odd_extension(w, grid, h):
    def gg(u):
        return torch.where(u == 0, 0.0, u * torch.log(torch.where(u == 0, 1.0, u.abs())))

    u = w[:, None] - grid[None, :]
    k = (gg(u + h) - 2.0 * gg(u) + gg(u - h)) / h / math.pi
    k[:, 0] = 0.0
    return k


def test_first_moment_sum_rule(limno2):
    sc, fc, fc3 = limno2
    ph = _spec(fc, sc, fc3)
    mesh = (2, 2, 2)
    q = [[0.5, 0.0, 0.0], [0.5, 0.5, 0.5]]
    r = ph.spectral_function(mesh, q, [300.0], frequency_points=[0.0])
    grid_np = r["self_energy_points"]
    h = grid_np[1] - grid_np[0]
    grid = torch.as_tensor(grid_np)
    omega = np.linspace(0.0, grid_np[-1] + h, 400_001)
    gamma = torch.as_tensor(r["gamma"][0]).reshape(-1, len(grid_np))  # [Q 3n, M]
    nu = torch.as_tensor(r["frequencies"]).reshape(-1)
    rules = {}
    for name, fn in (("closed form", _hilbert_matrix), ("Delta flipped", lambda *a: -_hilbert_matrix(*a)),
                     ("no odd extension", _no_odd_extension)):
        a, g, d = _a_from(gamma, nu, omega, grid, h, fn)
        moment = torch.trapezoid(torch.as_tensor(omega) * a, torch.as_tensor(omega), dim=-1)
        den = torch.as_tensor(omega) ** 2 - nu[:, None] ** 2 - 2 * nu[:, None] * d
        # poles A does not hold: a zero of the denominator where Gamma = 0, or one on the imaginary axis (the
        # denominator at w = 0, -nu^2 - 2 nu Delta(0), is then >= 0: the coupling is too strong for a stable mode)
        cross = (den[:, 1:] * den[:, :-1] <= 0) & ((g[:, 1:] == 0) | (g[:, :-1] == 0))
        rules[name] = (moment, cross.any(1) | (den[:, 0] >= 0))
    moment, pole = rules["closed form"]
    checked = (nu >= CUT) & ~pole
    err = float(((moment - nu).abs() / nu.clamp_min(CUT))[checked].max())
    errs = {k: float(((m - nu).abs() / nu.clamp_min(CUT))[checked & ~p].max()) for k, (m, p) in rules.items()}
    print(f"LiMnO2 2x1x1, random fc3, 2^3, 300 K: first moment vs nu over {int(checked.sum())} modes (skipped "
          f"{int(((nu >= CUT) & pole).sum())} with an undamped pole): {errs}")
    assert checked.sum() >= 20
    assert err <= 1e-8
    assert errs["Delta flipped"] > 1e-2 and errs["no odd extension"] > 1e-2
    # the method's own A on its report grid is the same function
    r2 = ph.spectral_function(mesh, q, [300.0], frequency_points=omega[::400])
    a_own = _a_from(gamma, nu, omega[::400], grid, h, _hilbert_matrix)[0].reshape(r2["spectral_function"][0].shape)
    assert np.abs(r2["spectral_function"][0] - a_own.numpy()).max() <= 1e-12 * np.abs(a_own.numpy()).max()


def test_weak_coupling_limit(limno2):
    sc, fc, fc3 = limno2
    mesh, q, temps = (2, 2, 2), [0.5, 0.5, 0.0], [300.0]
    base = _spec(fc, sc, fc3).spectral_function(mesh, q, temps, frequency_points=[1.0])
    nu = base["frequencies"]
    g_nu = np.array([np.interp(v, base["self_energy_points"], base["gamma"][0, i]) for i, v in enumerate(nu)])
    modes = np.nonzero((nu >= CUT) & (g_nu > 1e-3 * g_nu.max()))[0]
    errs = []
    for s in (3e-2, 3e-3):
        x = np.linspace(-6.0, 6.0, 241)
        r = _spec(fc, sc, s * fc3).spectral_function(mesh, q, temps, frequency_points=[1.0])
        assert np.abs(r["gamma"] - s * s * base["gamma"]).max() <= 1e-12 * s * s * np.abs(base["gamma"]).max()
        assert np.abs(r["delta"] - s * s * base["delta"]).max() <= 1e-12 * s * s * np.abs(base["delta"]).max()
        assert np.abs(r["frequency_shifts"] - s * s * base["frequency_shifts"]).max() <= (
            1e-12 * s * s * np.abs(base["frequency_shifts"]).max())
        worst = 0.0
        for i in modes:
            gam, shift = s * s * g_nu[i], r["frequency_shifts"][0, i]
            pts = nu[i] + shift + gam * x
            a = _spec(fc, sc, s * fc3).spectral_function(mesh, q, temps, frequency_points=pts)["spectral_function"]
            lor = gam / math.pi / ((pts - nu[i] - shift) ** 2 + gam * gam)
            worst = max(worst, np.abs(a[0, i] - lor).max() / lor.max())
        errs.append(worst)
    print(f"LiMnO2 2x1x1, random fc3 x s, {len(modes)} modes: max |A - Lorentzian| / peak {errs} at s = 3e-2, 3e-3")
    assert errs[1] < errs[0] / 10 and errs[1] <= 1e-2


def test_chunking_temperatures_and_errors(limno2):
    sc, fc, fc3 = limno2
    ph = _spec(fc, sc, fc3)
    mesh, q = (2, 2, 2), [[0.0, 0.0, 0.0], [0.5, 0.0, 0.5]]
    temps = [0.0, 300.0, 1000.0]
    r = ph.spectral_function(mesh, q, temps, self_energy_points=51)
    assert r["gamma"].shape == (3, 2, 24, 51) and r["spectral_function"].shape == (3, 2, 24, 2001)
    assert r["frequency_shifts"].shape == (3, 2, 24) and r["frequency_points"].shape == (2001,)
    assert np.all(r["gamma"][:, 0, :3] == 0) and np.all(r["spectral_function"][:, 0, :3] == 0)
    assert np.all(r["gamma"][:, :, :, 0] == 0) and np.all(r["gamma"][0] >= 0)
    one = ph.spectral_function(mesh, q[1], [300.0], self_energy_points=51)
    assert one["gamma"].shape == (1, 24, 51) and one["frequencies"].shape == (24,)
    for k in ("gamma", "delta", "spectral_function", "frequency_shifts"):
        assert np.abs(one[k][0] - r[k][1, 1]).max() <= 1e-14 * np.abs(r[k][1]).max(), k
    ph.ph3_chunk_bytes = 1  # one q1 per call
    r1 = ph.spectral_function(mesh, q, temps, self_energy_points=51)
    errs = {k: np.abs(r1[k] - r[k]).max() / np.abs(r[k]).max() for k in ("gamma", "delta", "spectral_function")}
    print(f"LiMnO2 2x1x1, random fc3, 2^3: one q1 per call vs one chunk {errs}")
    assert max(errs.values()) <= 1e-13
    for bad in (2, 3.0, True, "201"):
        with pytest.raises(ValueError, match="self_energy_points"):
            ph.spectral_function(mesh, q, temps, self_energy_points=bad)
    for bad in ([-1.0, 2.0], [float("nan")], [], [[float("inf")]]):
        with pytest.raises(ValueError, match="frequency_points"):
            ph.spectral_function(mesh, q, temps, frequency_points=bad)
    with pytest.raises(ValueError, match="temperatures"):
        ph.spectral_function(mesh, q, [-1.0])
    with pytest.raises(ValueError, match="temperatures"):
        ph.spectral_function(mesh, q, None)
    with pytest.raises(ValueError, match="mesh"):
        ph.spectral_function(mesh, [0.25, 0, 0], [300.0])
    no3 = Phonons(fc, sc, device="cpu", kernels=SpectralFunctionSpecKernels())
    with pytest.raises(ValueError, match="third_order=True"):
        no3.spectral_function(mesh, q, [300.0])


def test_chunk_limit_matches_header():
    from chgnet_b200 import _lib

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "chgnet_b200.h")).read(), flags=re.S)
    assert _lib.SE_MAX_CHUNKS == int(re.search(r"#define CHG_SE_MAX_CHUNKS\s+(\d+)", src).group(1))
