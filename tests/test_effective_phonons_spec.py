"""CPU: effective force constants by stochastic sampling (``effective_force_constants``, DESIGN.md section 12.12)
through the fp64 specifications of the two kernels (tests/effective_phonons_kernels.py), with analytic potentials."""
import re

import numpy as np
import pytest
import torch
from scipy.optimize import brentq

from chgnet_b200 import _lib
from chgnet_b200.phonons import (DISPLACEMENT_A2_AMU_THZ, H_OVER_KB_K_PER_THZ, THZ_PER_SQRT_EV_A2_AMU, Phonons,
                                 _expand_compact, acoustic_sum_rule, effective_force_constants, make_supercell,
                                 sampling_modes, translation_table)
from chgnet_b200.dynamics import ATOMIC_MASSES, KB
from effective_cells import FCC_CONV, FCC_LATTICE, FCC_Z, HarmonicSurrogate, QuarticSprings, fcc_bonds, fcc_springs
from effective_phonons_kernels import EffectiveSpecKernels, normal_variates
from oracle.phonons import PhononSpecKernels
from phonon_cells import limno2_211


def _run(forces, sc, fc, t, **kw):
    return effective_force_constants(forces, sc, fc, t, kernels=EffectiveSpecKernels(), device="cpu", **kw)


def _perm_inv(sc):
    perm = translation_table(sc)
    inv = np.empty_like(perm)
    np.put_along_axis(inv, perm, np.arange(len(sc.z))[None].repeat(len(perm), 0), axis=1)
    return torch.as_tensor(inv.astype(np.int64))


def test_translation_table_maps_positions():
    """perm[l, j] sits at r_j + R_l modulo the supercell lattice, on a non-diagonal M; each row is a permutation."""
    sc = make_supercell([FCC_Z, FCC_Z], np.array([[0, 0, 0], [0.25, 0.25, 0.25]]), FCC_LATTICE, [[2, 1, 0], [0, 1, 1],
                                                                                                  [1, 0, 2]])
    perm = translation_table(sc)
    inv_m = np.linalg.inv(sc.matrix.astype(np.float64))
    for l, r in enumerate(sc.points):
        x = (sc.frac + r @ inv_m) % 1.0
        d = (sc.frac[perm[l]] - x + 0.5) % 1.0 - 0.5
        assert np.abs(d).max() < 1e-12
        assert sorted(perm[l]) == list(range(len(sc.z)))


@pytest.mark.parametrize("quantum,t,seed,mixing", [(True, 300.0, 0, 0.5), (False, 700.0, 3, 1.0), (True, 0.0, 11, 0.2)])
def test_harmonic_surrogate_is_recovered_limno2(weights030, quantum, t, seed, mixing):
    """One iteration on F = F_0 - Phi_sc u returns Phi (unequal masses, nonzero residual forces); sigma_a and u0 are
    rounding."""
    sc, _, fc = limno2_211(weights030)
    f0 = np.random.default_rng(1).normal(size=(len(sc.z), 3)) * 0.05
    out, info = _run(HarmonicSurrogate(sc, fc, f0), sc, fc, t, n_samples=30, n_iterations=1, mixing=mixing,
                     quantum=quantum, seed=seed, batch_size=8)
    ref = acoustic_sum_rule(fc, sc.p2s)[0]
    assert np.abs(out - ref).max() <= 1e-10 * np.abs(ref).max()
    assert info["history"][0]["max_change"] <= 1e-10 * np.abs(ref).max()
    assert info["sigma_a"] <= 1e-6  # the moment formula cancels to ~sqrt(eps)
    assert abs(info["u0"]) <= 1e-10
    assert set(info["history"][0]) == {"max_change", "n_imaginary", "sigma_a", "u0"}
    assert info["harmonic_force_constants"] is not None and info["temperature"] == t and info["quantum"] == quantum


@pytest.mark.parametrize("quantum,t", [(True, 300.0), (False, 50.0)])
def test_harmonic_surrogate_is_recovered_fcc_nondiagonal(quantum, t):
    sc, fc = fcc_springs(2 * FCC_CONV, 3.0)
    f0 = np.random.default_rng(2).normal(size=(len(sc.z), 3)) * 0.1
    out, info = _run(HarmonicSurrogate(sc, fc, f0), sc, fc, t, n_samples=5, n_iterations=1, quantum=quantum, seed=5,
                     batch_size=2)
    ref = acoustic_sum_rule(fc, sc.p2s)[0]
    assert np.abs(out - ref).max() <= 1e-10 * np.abs(ref).max()
    assert info["sigma_a"] <= 1e-6


def test_sampler_covariance_matches_thermal_displacements():
    """The exact covariance sum A^2 e e^T / m in the diagonal blocks equals U(T) on the matching mesh; the sampled
    covariance agrees within 5 standard errors."""
    n, t = 4, 300.0
    sc, fc = fcc_springs([n, n, n], 3.0)
    phi = torch.as_tensor(acoustic_sum_rule(fc, sc.p2s)[0])
    masses = ATOMIC_MASSES[sc.z - 1]
    nu, e, amp, n_imag = sampling_modes(_expand_compact(phi, _perm_inv(sc)), masses, t, quantum=True,
                                        frequency_floor=0.5)
    assert n_imag == 0 and np.sort(np.abs(nu.numpy()))[3] > 0.5  # the floor is inactive
    w = (e * amp[:, None]).numpy() / np.sqrt(np.repeat(masses, 3))[None, :]  # rows A e / sqrt m
    cov = w.T @ w
    u_ref = Phonons(fc, sc, device="cpu", kernels=PhononSpecKernels()).thermal_displacement_matrices([n] * 3, [t])
    for j in range(len(sc.z)):
        assert np.abs(cov[3 * j : 3 * j + 3, 3 * j : 3 * j + 3] - u_ref["cartesian"][0, 0]).max() <= 1e-12 * cov.max()
    m = 400
    k = EffectiveSpecKernels()
    frac = torch.empty(m * len(sc.z), 3, dtype=torch.float32)
    u = torch.empty(m, len(sc.z), 3, dtype=torch.float64)
    lat = torch.as_tensor(sc.lattice)
    k.sample_displacements(e, amp, torch.as_tensor(1 / np.sqrt(masses)), torch.as_tensor(sc.frac), lat,
                           torch.linalg.inv(lat), 7, 0, 0, frac, u)
    x = u.reshape(m, -1).numpy()
    sampled = x.T @ x / m
    se = np.sqrt((np.diag(cov)[:, None] * np.diag(cov)[None, :] + cov**2) / m)
    assert np.abs(sampled - cov).max() <= 5 * se.max()


def _s2(k_eff, sc, bonds, t, quantum):
    """<s^2> of one bond under the sampling distribution of springs k_eff, from a numpy eigendecomposition."""
    _, fc = fcc_springs(sc.matrix, k_eff)
    n = len(sc.z)
    phi = _expand_compact(torch.as_tensor(acoustic_sum_rule(fc, sc.p2s)[0]), _perm_inv(sc)).numpy()
    m = ATOMIC_MASSES[FCC_Z - 1]
    lam, e = np.linalg.eigh(phi / m)
    nu = np.abs(np.sign(lam) * np.sqrt(np.abs(lam)) * THZ_PER_SQRT_EV_A2_AMU)
    if quantum:
        a2 = DISPLACEMENT_A2_AMU_THZ / nu / np.tanh(H_OVER_KB_K_PER_THZ * nu / (2 * t))
    else:
        a2 = KB * t * (THZ_PER_SQRT_EV_A2_AMU / nu) ** 2
    a2[np.argsort(nu)[:3]] = 0.0
    cov = (e * a2[None, :]) @ e.T / m
    i, j, eh = bonds
    c = cov.reshape(n, 3, n, 3)
    s2 = [eh[b] @ (c[i[b], :, i[b]] + c[j[b], :, j[b]] - c[i[b], :, j[b]] - c[j[b], :, i[b]]) @ eh[b]
          for b in range(len(i))]
    return float(np.mean(s2))


@pytest.mark.parametrize("quantum,t", [(False, 300.0), (True, 300.0)])
def test_quartic_springs_closed_form(quantum, t):
    """fcc springs k with a quartic bond term lam/4 s^4 converge to k_eff = k + 3 lam <s^2>(k_eff); u0 per cell is
    6 (-3/4) lam <s^2>^2; sigma_a is the residual norm of the stored samples."""
    k, lam = 3.0, 40.0
    sc = make_supercell([FCC_Z], np.zeros((1, 3)), FCC_LATTICE, 2 * FCC_CONV)
    bonds = fcc_bonds(sc)
    k_eff = brentq(lambda x: x - k - 3 * lam * _s2(x, sc, bonds, t, quantum), k, 3 * k)
    s2 = _s2(k_eff, sc, bonds, t, quantum)
    _, fc0 = fcc_springs(sc.matrix, k)
    pot = QuarticSprings(sc, k, lam, keep=True)
    n_samples = 256
    out, info = _run(pot, sc, fc0, t, n_samples=n_samples, n_iterations=6, mixing=1.0, quantum=quantum, seed=3,
                     batch_size=64)
    _, fc_eff = fcc_springs(sc.matrix, k_eff)
    i, j, eh = bonds
    nn = j[i == 0]
    k_fit = np.mean([-eh[b] @ out[0, j[b]] @ eh[b] for b in np.nonzero(i == 0)[0]])
    assert abs(k_fit - k_eff) <= 0.02 * k_eff, (k_fit, k_eff)
    assert np.abs(out - fc_eff).max() <= 0.05 * k_eff
    assert abs(info["u0"] - 6 * (-0.75) * lam * s2**2) <= 0.1 * abs(6 * 0.75 * lam * s2**2), (info["u0"], s2)
    # sigma_a from the last iteration's stored samples (mixing 1: the result is that iteration's fit)
    phi_sc = _expand_compact(torch.as_tensor(out), _perm_inv(sc)).numpy()
    f0 = pot.calls[0][1][0]
    ref = np.asarray(sc.frac, dtype=np.float32).astype(np.float64)
    num = den = 0.0
    for x, f in pot.calls[-(n_samples // 64):]:
        u = ((x - ref[None]) @ sc.lattice).reshape(len(x), -1)
        df = (f - f0[None]).reshape(len(x), -1)
        num += ((df + u @ phi_sc.T) ** 2).sum()
        den += (df**2).sum()
    assert abs(info["sigma_a"] - np.sqrt(num / den)) <= 1e-8, (info["sigma_a"], np.sqrt(num / den))
    assert info["sigma_a"] > 0.01
    assert len(nn) == 6


def test_moments_are_bitwise_independent_of_call_splits():
    """The spec moments over 1, 2 and 7 calls are bitwise equal, and equal a plain loop over the full supercell."""
    sc, fc = fcc_springs(2 * FCC_CONV, 3.0)
    n = len(sc.z)
    rng = np.random.default_rng(4)
    m = 7
    u = torch.as_tensor(rng.normal(size=(m, n, 3)))
    f = torch.as_tensor(rng.normal(size=(m, n, 3)))
    f0 = torch.as_tensor(rng.normal(size=(n, 3)))
    perm = torch.as_tensor(translation_table(sc))
    accs = []
    for parts in ([7], [3, 4], [1] * 7):
        acc = torch.zeros(18 * n + 2, dtype=torch.float64)
        s0 = 0
        for p in parts:
            EffectiveSpecKernels().displacement_moments(u[s0 : s0 + p], f[s0 : s0 + p], f0, perm, acc)
            s0 += p
        accs.append(acc)
    assert torch.equal(accs[0], accs[1]) and torch.equal(accs[0], accs[2])
    g = np.zeros((3, n, 3))
    b = np.zeros((3, n, 3))
    p = perm.numpy()
    for s in range(m):
        for l in range(len(p)):
            for jj in range(n):
                g[:, jj, :] += np.outer(u[s, p[l, 0]].numpy(), u[s, p[l, jj]].numpy())
                b[:, jj, :] += np.outer((f[s, p[l, 0]] - f0[p[l, 0]]).numpy(), u[s, p[l, jj]].numpy())
    a = accs[0].numpy()
    assert np.allclose(a[: 9 * n], g.reshape(-1), rtol=0, atol=1e-12)
    assert np.allclose(a[9 * n : 18 * n], b.reshape(-1), rtol=0, atol=1e-12)
    assert np.isclose(a[-2], float(((f - f0[None]) ** 2).sum()), rtol=1e-14)
    assert np.isclose(a[-1], float((f0[None] * u).sum()), rtol=1e-14)


def test_samples_are_a_function_of_seed_and_counter():
    """Two runs with one seed are bitwise equal, another seed differs; the variates do not depend on the chunking and
    are standard normal."""
    sc, fc = fcc_springs(2 * FCC_CONV, 3.0)
    pot = QuarticSprings(sc, 3.0, 40.0)
    a = _run(pot, sc, fc, 300.0, n_samples=8, n_iterations=2, seed=9, batch_size=3)
    b = _run(pot, sc, fc, 300.0, n_samples=8, n_iterations=2, seed=9, batch_size=3)
    c = _run(pot, sc, fc, 300.0, n_samples=8, n_iterations=2, seed=10, batch_size=3)
    assert np.array_equal(a[0], b[0]) and a[1]["history"] == b[1]["history"]
    assert not np.array_equal(a[0], c[0])
    x = normal_variates(5, 2, np.arange(10), 6)
    assert np.array_equal(x[4:7], normal_variates(5, 2, [4, 5, 6], 6))
    z = normal_variates(0, 0, np.arange(2000), 50).reshape(-1)
    assert abs(z.mean()) < 5 / np.sqrt(z.size) and abs(z.var() - 1) < 5 * np.sqrt(2 / z.size)


@pytest.mark.parametrize("kw", [dict(temperature=-1.0), dict(temperature=float("nan")), dict(temperature=np.inf),
                                dict(temperature=0.0, quantum=False), dict(n_iterations=0), dict(mixing=0.0),
                                dict(mixing=1.5), dict(frequency_floor=0.0), dict(batch_size=0), dict(n_samples=2),
                                dict(seed=-1)])
def test_bad_arguments_raise_before_any_force_call(kw):
    sc, fc = fcc_springs(2 * FCC_CONV, 3.0)  # 32 atoms in 32 cells: 3N - 3 = 93 needs n_samples >= 3

    def forces(frac):
        raise AssertionError("forces called")

    args = dict(temperature=300.0)
    args.update(kw)
    t = args.pop("temperature")
    with pytest.raises(ValueError):
        _run(forces, sc, fc, t, **args)


def test_scratch_helpers():
    src = open(_lib.__file__.replace("chgnet_b200/_lib.py", "include/chgnet_b200.h")).read()
    assert re.search(r"at least n_samples n_modes doubles", src)
    assert re.search(r"at least \(1 \+ n_samples\) \(18 n_prim N \+ 2\) doubles", src)
    assert _lib.sampler_scratch_doubles(5, 12) == 60
    assert _lib.moments_scratch_doubles(5, 2, 8) == 6 * (18 * 2 * 8 + 2)
