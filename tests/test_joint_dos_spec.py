"""CPU (fp64): two-phonon joint densities of states of chgnet_b200.phonons (``Phonons.joint_dos``,
``Phonons.phase_space``) with the specification of ``chg_joint_dos`` (oracle/phonons.py).

* the specification against a plain loop over (q1, tetrahedron, band pair, term), with negative frequencies, values
  below and on the cutoff, tied corner values, frequency points on corner values and T = 0;
* sum rules: the integral over w of D2(2) and D2(1) is 1/N and 2/N times the number of unmasked (q1, l1, l2);
* identities: the two class-1 terms agree, D2(q) = D2(-q), N2 at T = 0, and phase_space against joint_dos;
* a simple cubic spring crystal (three 1D chains, also tethered by an on-site spring): D2 and N2 against a
  Monte-Carlo histogram over continuous q1, with an error that falls with the mesh; the classical limit of N2 / T;
* the host path: chunking, n_imaginary, bad q-points and temperatures."""
import itertools

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import H_OVER_KB_K_PER_THZ, THERMAL_CUTOFF_THZ, gamma_mesh, tetrahedra
from oracle.phonon_dos import tetrahedron_weights
from oracle.phonons import PhononSpecKernels
from phonon_cells import limno2_211_spec, spec_phonons

CUT = THERMAL_CUTOFF_THZ
f64 = torch.float64


def _occ(nu, t):
    return 0.0 if t == 0 else 1.0 / np.expm1(H_OVER_KB_K_PER_THZ * nu / t)


def _loop(freqs, mesh, tets, target, omega, factors):
    """[len(factors), 3, F] by a plain loop over (q1 cell, tetrahedron, l1, l2, term): the three terms
    (nu2 - nu1, nu1 - nu2, nu1 + nu2), each corner weighted by ``factor(term, nu1, nu2)`` where both are >= the cutoff,
    every tetrahedron by 1 / (6 N)."""
    n1, n2, n3 = mesh
    n_q, nb = freqs.shape
    tq = np.array([target // (n2 * n3), (target // n3) % n2, target % n3])
    out = np.zeros((len(factors), 3, len(omega)))
    w = torch.as_tensor(omega, dtype=f64)
    for cell in itertools.product(range(n1), range(n2), range(n3)):
        for t in tets:
            c1 = (np.array(cell) + t) % mesh
            c2 = (tq - c1) % mesh
            q1 = (c1[:, 0] * n2 + c1[:, 1]) * n3 + c1[:, 2]
            q2 = (c2[:, 0] * n2 + c2[:, 1]) * n3 + c2[:, 2]
            for l1, l2 in itertools.product(range(nb), range(nb)):
                a, b = freqs[q1, l1], freqs[q2, l2]
                m = (a >= CUT) & (b >= CUT)
                for term, f in enumerate((b - a, a - b, a + b)):
                    order = np.argsort(f, kind="stable")
                    wt = tetrahedron_weights(torch.as_tensor(f[order]).expand(len(omega), 4), w)[2].numpy()
                    for s, fac in enumerate(factors):
                        c = np.array([fac(term, a[i], b[i]) if m[i] else 0.0 for i in range(4)])
                        out[s, term] += wt @ c[order]
    return out / (6.0 * n_q)


def _d2_factor(term, a, b):
    return 1.0


def _n2_factor(t):
    def fac(term, a, b):
        na, nb = _occ(a, t), _occ(b, t)
        return (na - nb, nb - na, na + nb + 1.0)[term]
    return fac


def _random_freqs(n_q, nb, rng, grid=None):
    nu = rng.uniform(-1.0, 6.0, size=(n_q, nb))
    nu[::4, 0] = 0.0
    nu[1::4, 0] = 5e-4
    nu[2::4, 0] = CUT
    nu[3::4, 0] = -2e-2
    if grid is not None:
        nu = np.round(nu / grid) * grid
    return np.sort(nu, axis=1)


def _terms(freqs, mesh, targets, omega, temps, tets=None):
    tets = tetrahedra(mesh, np.eye(3)) if tets is None else tets
    om = torch.as_tensor(np.broadcast_to(omega, (len(targets), len(omega))).copy())
    return PhononSpecKernels().joint_dos_terms(
        torch.as_tensor(freqs), mesh, torch.as_tensor(tets), torch.as_tensor(np.asarray(targets, dtype=np.int32)), om,
        None if temps is None else torch.as_tensor(np.asarray(temps, dtype=np.float64)), CUT).numpy()


@pytest.mark.parametrize("grid", [None, 0.5], ids=["random", "ties_on_a_grid"])
def test_spec_matches_plain_loop(grid):
    rng = np.random.default_rng(1 if grid is None else 2)
    mesh = (3, 3, 3)
    freqs = _random_freqs(27, 3, rng, grid)
    temps = [0.0, 300.0, 1000.0]
    omega = np.concatenate([np.linspace(-3.0, 12.0, 31), np.arange(-2.0, 12.5, 0.5), [CUT, 0.0]])  # grid: on vertices
    targets = [0, 14, 22]
    got = _terms(freqs, mesh, targets, omega, temps)  # [Q, 1 + T, 3, F]
    tets = tetrahedra(mesh, np.eye(3))
    for i, tq in enumerate(targets):
        want = _loop(freqs, mesh, tets, tq, omega, [_d2_factor] + [_n2_factor(t) for t in temps])
        err = np.abs(got[i] - want).max() / np.abs(want).max()
        assert err <= 1e-13, (tq, err)
    out = torch.empty(len(targets), 1 + len(temps), 2, len(omega), dtype=f64)
    PhononSpecKernels().joint_dos(torch.as_tensor(freqs), mesh, torch.as_tensor(tets),
                                  torch.as_tensor(np.asarray(targets, dtype=np.int32)),
                                  torch.as_tensor(np.broadcast_to(omega, (3, len(omega))).copy()),
                                  torch.as_tensor(temps), CUT, out)
    assert np.array_equal(out[:, :, 0].numpy(), got[:, :, 0] + got[:, :, 1])
    assert np.array_equal(out[:, :, 1].numpy(), got[:, :, 2])
    # the two class-1 terms are one sum mapped by q1 -> q - q1, l1 <-> l2 (the kernel evaluates one and doubles it)
    scale = np.abs(got).max()
    assert np.abs(got[:, :, 0] - got[:, :, 1]).max() <= 1e-12 * scale
    # at T = 0: N2(2) = D2(2), N2(1) = 0
    assert np.abs(got[:, 1, 2] - got[:, 0, 2]).max() <= 1e-12 * scale
    assert np.abs(got[:, 1, :2]).max() <= 1e-12 * scale


def test_class1_terms_agree_on_a_skewed_mesh():
    rng = np.random.default_rng(4)
    mesh = (2, 3, 4)
    freqs = _random_freqs(24, 4, rng)
    lat = graphgen.limno2_structure()[2]
    for d in range(4):
        got = _terms(freqs, mesh, range(24), np.linspace(-6, 12, 37), [0.0, 500.0], tetrahedra(mesh, lat, d))
        assert np.abs(got[:, :, 0] - got[:, :, 1]).max() <= 1e-12 * np.abs(got).max()


@pytest.mark.parametrize("masked", [False, True])
def test_integral_sum_rule(masked):
    """int D2(2) dw = (1/N) #{unmasked (q1, l1, l2)}, int D2(1) dw = twice that: each mesh point is a corner of 24
    tetrahedra and each corner weight integrates to 1/4.  The densities are piecewise cubic between the sorted corner
    values: 3-point Gauss-Legendre between consecutive values is exact."""
    rng = np.random.default_rng(8)
    mesh, nb = (2, 2, 2), 3
    freqs = np.sort(rng.uniform(0.5, 6.0, size=(8, nb)), axis=1)
    if masked:
        freqs[3, 0] = -0.7
        freqs[5, :2] = [0.0, 5e-4]
    target = 5
    q = gamma_mesh(mesh)
    q2 = np.round((q[target] - q) * np.array(mesh)).astype(int) % mesh
    i2 = (q2[:, 0] * 2 + q2[:, 1]) * 2 + q2[:, 2]
    a, b = freqs[:, :, None], freqs[i2][:, None, :]
    knots = np.unique(np.concatenate([(a + b).ravel(), (b - a).ravel(), (a - b).ravel()]))
    x, gw = np.polynomial.legendre.leggauss(3)
    pts = (0.5 * np.diff(knots)[:, None] * x + 0.5 * (knots[1:] + knots[:-1])[:, None]).ravel()
    wts = (0.5 * np.diff(knots)[:, None] * gw).ravel()
    got = _terms(freqs, mesh, [target], pts, None)[0, 0]  # [3, F]
    n_kept = ((a >= CUT) & (b >= CUT)).sum()
    if not masked:
        assert n_kept == 8 * nb * nb
    assert abs(got[2] @ wts - n_kept / 8) <= 1e-13 * nb * nb
    assert abs((got[0] + got[1]) @ wts - 2 * n_kept / 8) <= 1e-13 * nb * nb


def test_time_reversal():
    """nu(-q) = nu(q) and the 6-tetrahedron set is inversion symmetric: D2(q) = D2(-q), N2 too."""
    rng = np.random.default_rng(6)
    mesh = (4, 4, 3)
    q = gamma_mesh(mesh)
    mi = np.round(-q * np.array(mesh)).astype(int) % mesh
    minus = (mi[:, 0] * 4 + mi[:, 1]) * 3 + mi[:, 2]
    r = rng.uniform(-0.5, 4.0, size=(48, 4))
    freqs = np.sort(r + r[minus], axis=1)
    targets = [1, 5, 17, 31]
    omega = np.linspace(0, 16, 41)
    a = _terms(freqs, mesh, targets, omega, [0.0, 300.0])
    b = _terms(freqs, mesh, [int(minus[t]) for t in targets], omega, [0.0, 300.0])
    assert all(minus[t] != t for t in targets)
    assert np.abs(a - b).max() <= 1e-12 * np.abs(a).max()


def _chain_freqs(q, nu0=0.0):
    """Branch values sqrt(nu0^2 + NU_MAX^2 sin^2 pi q_a) [..., 3]: the three chains, tethered by an on-site spring
    when nu0 > 0 (a gap: the occupations stay bounded)."""
    return np.sqrt(nu0**2 + (NU_MAX * np.sin(np.pi * q)) ** 2)


NU_MAX = 6.0  # THz


@pytest.mark.parametrize("nu0", [0.0, 2.0], ids=["chains", "tethered_chains"])
def test_monte_carlo_convergence(nu0):
    """D2 (and N2 at 300 K for the tethered chains) of the three-chain crystal at two q against a 10^6-sample
    histogram over continuous q1 (bin averages, 4 midpoints per bin).  N2 of the untethered chains diverges
    logarithmically (n ~ k T / h nu on the planes where a branch vanishes), so it is only checked with the gap."""
    rng = np.random.default_rng(12)
    targets = np.array([[0.5, 0.25, 0.125], [0.375, 0.125, 0.25]])
    temp = 300.0
    n_bins, sub = 24, 4
    edges = np.linspace(0.0, 2 * np.hypot(nu0, NU_MAX), n_bins + 1)
    h = edges[1] - edges[0]
    omega = (edges[:-1, None] + h * (np.arange(sub) + 0.5)[None, :] / sub).ravel()
    q1 = rng.uniform(size=(10**6, 3))
    slots = 2 if nu0 > 0 else 1
    errs = {}
    for ti, tq in enumerate(targets):
        a, b = _chain_freqs(q1, nu0), _chain_freqs(tq - q1, nu0)  # [S, 3]: branch values at q1 and q - q1
        a, b = np.repeat(a, 3, axis=1), np.tile(b, 3)  # all 9 (branch, branch) pairs
        keep = (a >= CUT) & (b >= CUT)
        na, nb = _occ(np.where(keep, a, 1.0), temp), _occ(np.where(keep, b, 1.0), temp)
        mc = np.zeros((2, 2, n_bins))  # [slot, class, bin]
        for s, (w1, w2) in enumerate([(1.0, 1.0), (na - nb, na + nb + 1.0)][:slots]):
            # class 1: d(w + nu1 - nu2) with (n1 - n2), d(w - nu1 + nu2) with -(n1 - n2) (D2: both with 1)
            w1 = np.where(keep, w1, 0.0) * np.ones_like(a)
            w2 = np.where(keep, w2, 0.0) * np.ones_like(a)
            mc[s, 0] = (np.histogram((b - a).ravel(), edges, weights=w1.ravel())[0]
                        + np.histogram((a - b).ravel(), edges, weights=(-w1 if s else w1).ravel())[0])
            mc[s, 1] = np.histogram((a + b).ravel(), edges, weights=w2.ravel())[0]
        mc /= len(q1) * h
        for n in (8, 16, 24):
            mesh = (n, n, n)
            freqs = np.sort(_chain_freqs(gamma_mesh(mesh), nu0), axis=1)
            idx = np.round(tq * n).astype(int) % n
            t = _terms(freqs, mesh, [(idx[0] * n + idx[1]) * n + idx[2]], omega, [temp])[0]  # [2, 3, F]
            tet = np.stack([t[:, 0] + t[:, 1], t[:, 2]], 1).reshape(2, 2, n_bins, sub).mean(-1)
            for s in range(slots):
                for c in range(2):
                    errs.setdefault((ti, s, c), []).append(np.abs(tet[s, c] - mc[s, c]).mean() / np.abs(mc[s, c]).max())
    for key, e in errs.items():
        print(f"nu0 {nu0}, target {key[0]}, {'D2' if key[1] == 0 else 'N2 300 K'}, class {key[2] + 1}: mean "
              f"|tetrahedron - MC| / max over bins, meshes 8, 16, 24: " + ", ".join(f"{x:.2e}" for x in e))
    # calibrated on these models (largest at 24^3: 0.050 for the chains, 0.035 with the gap).  The sorted bands
    # cross all over the zone, and the error of interpolating them across crossings is not monotone from 16^3 to 24^3
    # with the gap (it falls from 8^3 on in every case)
    for key, e in errs.items():
        assert e[1] < e[0] and e[2] < e[0], key
        assert e[2] <= (0.06 if nu0 == 0 else 0.04), key


def test_classical_limit():
    """N2 / T tends to the sum with n -> k T / (h nu): the gap falls as (h nu_max / k T)^2."""
    rng = np.random.default_rng(3)
    mesh = (3, 3, 3)
    freqs = np.sort(rng.uniform(0.2, NU_MAX, size=(27, 2)), axis=1)
    freqs[0] = 0.0
    omega = np.linspace(0.0, 2 * NU_MAX, 25)
    tets = tetrahedra(mesh, np.eye(3))
    temps = [2000.0, 4000.0, 8000.0]
    got = _terms(freqs, mesh, [4], omega, temps)[0]  # [1 + T, 3, F]

    def classical(term, a, b):  # k T / h (1 / nu), divided by T
        ia, ib = 1.0 / (H_OVER_KB_K_PER_THZ * a), 1.0 / (H_OVER_KB_K_PER_THZ * b)
        return (ia - ib, ib - ia, ia + ib)[term]

    want = _loop(freqs, mesh, tets, 4, omega, [classical])[0]
    gaps = []
    for i, t in enumerate(temps):
        gaps.append(np.abs(got[1 + i] / t - want).max() / np.abs(want).max())
        assert gaps[-1] <= (H_OVER_KB_K_PER_THZ * NU_MAX / t) ** 2
    print("N2 / T against the classical limit at 2000, 4000, 8000 K:", gaps)
    assert 3.5 <= gaps[0] / gaps[1] <= 4.5 and 3.5 <= gaps[1] / gaps[2] <= 4.5


@pytest.fixture(scope="module")
def limno2_211(weights030):
    return limno2_211_spec(weights030)


def test_phase_space_equals_joint_dos_at_the_modes(limno2_211):
    ph = limno2_211
    mesh = (3, 2, 2)
    temps = [0.0, 300.0]
    ps = ph.phase_space(mesh, temps)
    nu = ps["frequencies"]
    n3 = nu.shape[1]
    assert ps["jdos"].shape == (12, n3, 2) and ps["weighted_jdos"].shape == (2, 12, n3, 2)
    assert (nu[0, np.argsort(np.abs(nu[0]), kind="stable")[:3]] == 0).all() and (np.diff(nu, axis=1) >= 0).all()
    kept = nu >= CUT
    assert (ps["jdos"][~kept] == 0).all() and (ps["weighted_jdos"][:, ~kept] == 0).all()
    scale = np.abs(ps["weighted_jdos"]).max()
    q = gamma_mesh(mesh)
    for i in (0, 1, 7, 11):
        jd = ph.joint_dos(mesh, q[i], nu[i], temps)
        want = np.where(kept[i][:, None], jd["jdos"].T, 0.0)
        assert np.abs(ps["jdos"][i] - want).max() <= 1e-12 * scale
        want_w = np.where(kept[i][None, :, None], jd["weighted_jdos"].transpose(0, 2, 1), 0.0)
        assert np.abs(ps["weighted_jdos"][:, i] - want_w).max() <= 1e-12 * scale
    assert np.allclose(ps["average_jdos"], ps["jdos"][kept].mean(0), rtol=1e-13, atol=0)
    assert np.allclose(ps["average_weighted_jdos"], ps["weighted_jdos"][:, kept].mean(1), rtol=1e-13, atol=0)
    # T = 0
    assert np.abs(ps["weighted_jdos"][0, :, :, 1] - ps["jdos"][:, :, 1]).max() <= 1e-12 * scale
    assert np.abs(ps["weighted_jdos"][0, :, :, 0]).max() <= 1e-12 * scale


def test_host_path(limno2_211):
    ph = limno2_211
    mesh = (3, 2, 2)
    temps = [0.0, 300.0, 1000.0]
    q = np.array([[0.0, 0.0, 0.0], [1 / 3, 0.5, 0.0], [-1 / 3, 1.5, 0.5]])
    jd = ph.joint_dos(mesh, q, temperatures=temps)
    ps = ph.phase_space(mesh, temps)
    assert jd["jdos"].shape == (3, 2, 201) and jd["weighted_jdos"].shape == (3, 3, 2, 201)
    w = jd["frequency_points"]
    assert w[0] == 0 and w[-1] == 2 * ps["frequencies"].max()
    small = spec_phonons(ph.force_constants, ph.cell)
    small.eigh_batch = 5
    small.jdos_chunk_bytes = 1  # one target per call
    jd2, ps2 = small.joint_dos(mesh, q, temperatures=temps), small.phase_space(mesh, temps)
    for a, b in ((jd, jd2), (ps, ps2)):
        for key in a:
            if isinstance(a[key], np.ndarray):
                assert np.abs(a[key] - b[key]).max() <= 1e-13 * max(np.abs(a[key]).max(), 1e-300), key
    n_imag = ph.thermal_properties(mesh, [300.0])["n_imaginary"]
    assert n_imag > 0 and jd["n_imaginary"] == n_imag and ps["n_imaginary"] == n_imag
    # q2 = -q1 on the mesh: the target -1/3 equals 2/3, 1.5 equals 0.5
    assert np.array_equal(jd["jdos"][2], ph.joint_dos(mesh, [2 / 3, 0.5, 0.5])["jdos"])
    for bad in ([0.25, 0.0, 0.0], [np.nan, 0, 0], [0.0, 0.5 + 1e-6, 0.0]):
        with pytest.raises(ValueError):
            ph.joint_dos(mesh, bad)
    for bad in ([-1.0], [np.inf], [300.0, np.nan]):
        with pytest.raises(ValueError):
            ph.joint_dos(mesh, q, temperatures=bad)
        with pytest.raises(ValueError):
            ph.phase_space(mesh, bad)
