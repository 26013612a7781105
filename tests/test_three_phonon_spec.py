"""CPU (fp64): third-order force constants, three-phonon interaction strengths, linewidths and the RTA lattice thermal
conductivity of chgnet_b200.phonons with the specifications of ``chg_phonon_interaction`` and ``chg_imag_self_energy``
(tests/three_phonon_kernels.py).

* the closed form of P on a spring crystal with cubic terms on its three chains (constant, 1/N, masses, frequencies);
* P against the full supercell contraction on commensurate meshes (the image averages), and its independence of the
  G that reduces q2 (the Umklapp phase; its flipped sign fails);
* ``third_order_force_constants`` on an analytic model and against central differences of the fp64 oracle;
* the linewidth weights against the phase space of ``joint_dos``, a plain loop over (q1, tetrahedron, band pair),
  T = 0 and the classical limit;
* ``thermal_conductivity`` against its mode sum, chunking, and input errors; the header's chunk limit."""
import itertools
import math
import os
import re

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.dynamics import KB
from chgnet_b200.phonons import (DISPLACEMENT_A2_AMU_THZ, H_EV_PER_THZ, H_OVER_KB_K_PER_THZ, KAPPA_W_PER_MK,
                                 THERMAL_CUTOFF_THZ, Phonons, gamma_mesh, make_supercell,
                                 _degenerate_average, third_order_force_constants)
from oracle.hessian import oracle_hvp
from oracle.phonon_dos import tetrahedron_weights
from phonon_cells import CU, limno2_211, springs
from three_phonon_kernels import ThreePhononSpecKernels, interaction_strengths, vertex_weights

CUT = THERMAL_CUTOFF_THZ
f64 = torch.float64
KS = (3.0, 1.7, 4.4)
GC = (2.0, -1.3, 0.9)  # cubic coefficients of the three chains (eV/A^3)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _spec(fc, sc, fc3):
    return Phonons(fc, sc, fc3=fc3, device="cpu", kernels=ThreePhononSpecKernels())


def _chain_fc3(sc, g=GC):
    """Compact Phi3 [1, N, N, 3, 3, 3] of the potential sum_c g_c / 6 (u_l+1,c - u_l,c)^3 on the spring crystal."""
    n = len(sc.z)
    inv = np.linalg.inv(sc.lattice)
    out = np.zeros((1, n, n, 3, 3, 3))
    a = np.diag(sc.prim_lattice)
    for c in range(3):
        nb = {}
        for sgn in (1, -1):
            x = ((sgn * a[c] * np.eye(3)[c]) @ inv) % 1.0
            nb[sgn] = int(np.argmin(np.abs((sc.frac - x + 0.5) % 1.0 - 0.5).sum(1)))
        p, m = nb[1], nb[-1]
        for (j1, j2), v in {(0, p): 1, (p, 0): 1, (p, p): -1, (0, m): -1, (m, 0): -1, (m, m): 1}.items():
            out[0, j1, j2, c, c, c] += v * g[c]
    return out


def _spring_phonons(m=(3, 3, 3)):
    ph, nu_max = springs(m, ks=KS)
    return _spec(ph.force_constants, ph.cell, _chain_fc3(ph.cell)), nu_max


def _sets(nu, tol=1e-7):
    """Degenerate sets of the ascending nu [3n]: a list of index arrays."""
    cut = np.nonzero(np.abs(np.diff(nu)) > tol)[0] + 1
    return np.split(np.arange(len(nu)), cut)


def test_closed_form_spring_crystal():
    ph, nu_max = _spring_phonons()
    mesh = (4, 3, 5)
    n_mesh = int(np.prod(mesh))
    q_all = gamma_mesh(mesh)
    hbar, ev, amu = 6.62607015e-34 / (2 * np.pi), 1.602176634e-19, 1.66053906660e-27
    m_si = ph.masses[0] * amu
    worst, checked = 0.0, 0
    for q in (np.array([0.25, 1 / 3, 0.4]), np.array([0.5, 2 / 3, 0.8]), np.array([0.75, 0.0, 0.2])):
        p = ph._interaction_strength(mesh, q)  # [N, 3, 3, 3]
        for i1, q1 in enumerate(q_all):
            q2 = (q - q1) % 1.0
            qs = (q, q1, q2)
            branch = [nu_max * np.abs(np.sin(np.pi * x)) for x in qs]  # [3] per wave vector, branch c along axis c
            bands = [np.sort(b) for b in branch]
            want = np.zeros(3)
            for c in range(3):
                s = np.abs(np.sin(np.pi * q[c]) * np.sin(np.pi * q1[c]) * np.sin(np.pi * q2[c]))
                if min(b[c] for b in branch) < CUT:
                    continue
                want[c] = (hbar**3 * (GC[c] * ev / 1e-30) ** 2 * s
                           / (36 * n_mesh * (m_si * KS[c] * ev / 1e-20) ** 1.5) / ev**2)
            scale = want.max() if want.max() > 0 else 1.0
            for s0, s1, s2 in itertools.product(*(_sets(b) for b in bands)):
                got = p[i1][np.ix_(s0, s1, s2)].sum()
                br = [set(np.nonzero(np.abs(branch[k] - bands[k][s[0]]) <= 1e-7)[0]) for k, s in
                      enumerate((s0, s1, s2))]
                exp = sum(want[c] for c in br[0] & br[1] & br[2])
                worst = max(worst, abs(got - exp) / scale)
                checked += 1
    print(f"spring crystal with cubic chains: max |P - closed form| / max P = {worst:.2e} over {checked} set triples")
    assert worst <= 1e-12


def _translation_map(sc):
    """[n_cells, N]: the atom that atom j becomes when moved by the lattice point R_l."""
    inv_m = np.linalg.inv(sc.matrix.astype(np.float64))
    out = np.empty((len(sc.points), len(sc.z)), dtype=np.int64)
    for l, r in enumerate(sc.points):
        moved = (sc.frac + r @ inv_m) % 1.0
        d = np.abs((moved[:, None, :] - sc.frac[None, :, :] + 0.5) % 1.0 - 0.5).sum(2)
        out[l] = np.argmin(d, axis=1)
    return out


def _random_symmetric_fc3(sc, seed):
    """(full [3N, 3N, 3N], compact [n_prim, N, N, 3, 3, 3]) of a random fc3, periodic in the primitive lattice and
    symmetric under every permutation of its three (atom, axis) indices."""
    n, n_prim = len(sc.z), len(sc.p2s)
    n_cells = n // n_prim
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((n_prim, n, n, 3, 3, 3))
    tr = _translation_map(sc)
    full = np.zeros((n, n, n, 3, 3, 3))
    for k in range(n_prim):
        for l in range(n_cells):
            i = sc.p2s[k] + l  # atom k n_cells + l sits at r_k + R_l
            t = tr[l]
            full[np.ix_([i], t, t)] = base[k][None]
    full = full.transpose(0, 3, 1, 4, 2, 5).reshape(3 * n, 3 * n, 3 * n)
    full = sum(full.transpose(p) for p in itertools.permutations(range(3))) / 6
    compact = full.reshape(n, 3, n, 3, n, 3)[sc.p2s].transpose(0, 2, 4, 1, 3, 5)
    return full, np.ascontiguousarray(compact)


def _supercell_route(ph, full, mesh, target, q1):
    """P [3n, 3n, 3n] from the full supercell fc3 and the supercell normal modes e_k(q) e^{2 pi i q.r} / sqrt(N m)."""
    sc = ph.cell
    n_mesh = int(np.prod(mesh))
    pos = sc.frac @ sc.matrix  # primitive fractional coordinates of every supercell atom
    qs = [target, q1, (target - q1) % 1.0]
    nus, modes = ph.frequencies(np.array(qs), eigenvectors=True)
    us = []
    for q, e in zip(qs, modes):
        ph_ = np.exp(2j * np.pi * pos @ q)  # [N]
        u = e.reshape(len(sc.p2s), 3, -1)[sc.s2p] * (ph_ / np.sqrt(ph.masses[sc.s2p] * n_mesh))[:, None, None]
        us.append(u.reshape(-1, e.shape[1]))  # [3N, mode]
    t = np.einsum("ijk,il,jm,kn->lmn", full, us[0].conj(), us[1], us[2])
    nu = nus.copy()
    for k, q in enumerate(qs):  # the Gamma rule of the mesh frequencies
        if np.all(np.abs(q - np.round(q)) < 1e-12):
            nu[k, np.argsort(np.abs(nu[k]), kind="stable")[:3]] = 0.0
    keep = (nu[0] >= CUT)[:, None, None] & (nu[1] >= CUT)[None, :, None] & (nu[2] >= CUT)[None, None, :]
    den = nu[0][:, None, None] * nu[1][None, :, None] * nu[2][None, None, :]
    return np.where(keep, DISPLACEMENT_A2_AMU_THZ**3 / 36 * np.abs(t) ** 2 / np.where(keep, den, 1), 0.0)


def _set_sums(p, nus):
    """P summed over the degenerate sets of each of the three modes."""
    s = [_sets(x, 1e-6) for x in nus]
    return np.array([[[p[np.ix_(a, b, c)].sum() for c in s[2]] for b in s[1]] for a in s[0]])


@pytest.fixture(scope="module")
def limno2(weights030):
    sc, g, fc = limno2_211(weights030)
    return sc, g, fc


@pytest.mark.parametrize("cell", ["limno2_211", "springs_333"])
def test_supercell_route(cell, request):
    if cell == "limno2_211":
        sc, _, fc = request.getfixturevalue("limno2")
        mesh = (2, 1, 1)
    else:
        ph0, _ = springs((3, 3, 3), ks=KS)
        sc, fc, mesh = ph0.cell, ph0.force_constants, (3, 3, 3)
    full, compact = _random_symmetric_fc3(sc, seed=5)
    ph = _spec(fc, sc, compact)
    q_all = gamma_mesh(mesh)
    worst = 0.0
    for target in q_all[: 4]:
        p = ph._interaction_strength(mesh, target)
        for i1, q1 in enumerate(q_all):
            want = _supercell_route(ph, full, mesh, target, q1)
            nus = ph.frequencies(np.array([target, q1, (target - q1) % 1.0]))
            got_s, want_s = _set_sums(p[i1], nus), _set_sums(want, nus)
            worst = max(worst, np.abs(got_s - want_s).max() / max(np.abs(want_s).max(), 1e-300))
    print(f"{cell}: max |P - supercell contraction| / max = {worst:.2e}")
    assert worst <= 1e-12


def test_umklapp_phase(limno2):
    sc, _, fc = limno2
    _, compact = _random_symmetric_fc3(sc, seed=9)
    ph = _spec(fc, sc, compact)
    rng = np.random.default_rng(4)
    frac = torch.as_tensor(sc.prim_frac)
    args = (ph._fc3, ph._img_ptr, ph._img_vec, ph._s2p, ph._inv_sqrt_m, frac, 8, CUT)

    def p_at(q, q1, q2, sign=1.0):
        nu, e = ph.frequencies(np.array([q, q1, q2]), eigenvectors=True)
        e = torch.as_tensor(e).transpose(1, 2)  # mode-major
        nu = torch.as_tensor(nu)
        out = interaction_strengths(*args, torch.as_tensor(q), nu[0], e[0], torch.as_tensor(q1)[None], nu[1:2],
                                    e[1:2], torch.as_tensor(q2)[None], nu[2:3], e[2:3], phase_sign=sign)[0].numpy()
        return _set_sums(out, nu.numpy())

    worst, flipped = 0.0, 0.0
    for _ in range(4):
        q, q1 = rng.random(3), rng.random(3)
        red = (q - q1) % 1.0
        ref = p_at(q, q1, red)
        scale = np.abs(ref).max()
        for q2 in (q - q1, red + rng.integers(-2, 3, 3)):
            worst = max(worst, np.abs(p_at(q, q1, q2) - ref).max() / scale)
            flipped = max(flipped, np.abs(p_at(q, q1, q2, -1.0) - p_at(q, q1, red, -1.0)).max() / scale)
    print(f"LiMnO2 2x1x1: P with q2 reduced, unreduced and shifted by G agree to {worst:.2e}; with the phase's sign "
          f"flipped they differ by {flipped:.2e}")
    assert worst <= 1e-12
    assert flipped >= 1e-3


def test_extraction_analytic_chain():
    ph0, _ = springs((3, 3, 3), ks=KS)
    sc = ph0.cell
    n = len(sc.z)
    compact = _chain_fc3(sc)
    tr = _translation_map(sc)
    full = np.zeros((n, n, n, 3, 3, 3))
    for l in range(n):
        full[np.ix_([l], tr[l], tr[l])] = compact[0][None]
    full = full.transpose(0, 3, 1, 4, 2, 5).reshape(3 * n, 3 * n, 3 * n)
    h0 = np.zeros((n, 3, n, 3))
    fc = ph0.force_constants[0]
    for l in range(n):
        h0[l, :, tr[l]] = fc.transpose(0, 1, 2)
    h0 = h0.reshape(3 * n, 3 * n)

    def hvp_at(frac, v):
        d = (frac - sc.frac + 0.5) % 1.0 - 0.5
        u = (d @ sc.lattice).reshape(-1)
        h = h0 + np.einsum("ijk,k->ij", full, u)
        return (v.reshape(len(v), -1) @ h.T).reshape(v.shape)

    got = third_order_force_constants(hvp_at, sc, 0.03)
    err = np.abs(got - compact).max() / np.abs(compact).max()
    print(f"analytic chain model: max |Phi3 - exact| / max = {err:.2e}")
    assert err <= 1e-12
    for bad in (0.0, -0.01, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="displacement"):
            third_order_force_constants(hvp_at, sc, bad)


def test_extraction_against_oracle(weights030):
    sc = make_supercell(*CU, [2, 2, 2])
    n = len(sc.z)
    h = 0.03

    def hvp_at(frac, v):
        g = graphgen.make_crystal_graph(sc.z, frac, sc.lattice)
        k = v.shape[0]
        return oracle_hvp(weights030, [g] * k, torch.as_tensor(v.reshape(k * n, 3)), None).reshape(k, n, 3).numpy()

    got = third_order_force_constants(hvp_at, sc, h)
    # independent columns: a few (k, a) and directions j'' c by direct central differences
    worst = 0.0
    for a, col in ((0, 0), (1, 7), (2, 20)):
        hs = []
        for sgn in (1, -1):
            frac = sc.frac.copy()
            frac[sc.p2s[0]] += sgn * h * np.linalg.inv(sc.lattice)[a]
            v = np.zeros((1, n, 3))
            v.reshape(-1)[col] = 1.0
            hs.append(hvp_at(frac % 1.0, v)[0])
        want = (hs[0] - hs[1]) / (2 * h)  # [j', b] = d H[j' b, col] / d u
        worst = max(worst, np.abs(got[0, :, col // 3, a, :, col % 3] - want).max())
    scale = np.abs(got).max()
    asr = np.abs(got.sum(axis=2)).max() / scale
    print(f"Cu 2x2x2 through the oracle: max |Phi3 - central differences| = {worst:.2e} (max |Phi3| {scale:.3e}); "
          f"translational sum {asr:.2e} of max")
    assert worst <= 1e-12 * scale
    assert asr <= 1e-8


def _limno2_spec_ph(weights030, seed=3):
    sc, _, fc = limno2_211(weights030)
    _, compact = _random_symmetric_fc3(sc, seed)
    return _spec(fc, sc, compact)


def test_weights_reproduce_phase_space(limno2):
    sc, _, fc = limno2
    ph = _spec(fc, sc, np.zeros((len(sc.p2s), len(sc.z), len(sc.z), 3, 3, 3)))
    mesh = (3, 2, 2)
    temps = [0.0, 300.0, 1000.0]
    ps = ph.phase_space(mesh, temps)
    mesh_t, nu, _, _, tets, _ = ph._three_phonon_mesh(mesh, temps)
    n_mesh, nb = nu.shape
    t = torch.as_tensor(np.array(temps))
    worst = 0.0
    for target in range(n_mesh):
        p = torch.full((n_mesh, nb, nb, nb), 1.0 / n_mesh, dtype=f64)
        gamma = torch.zeros(len(temps), nb, dtype=f64)
        q1 = torch.arange(n_mesh, dtype=torch.int32)
        ph.kernels.imag_self_energy(nu, mesh_t, tets, target, nu[target].contiguous(), q1, p, t, CUT, gamma)
        want = 18 * math.pi / H_EV_PER_THZ**2 * ps["weighted_jdos"][:, target].sum(-1)  # [T, 3n]
        worst = max(worst, np.abs(gamma.numpy() - want).max() / np.abs(want).max())
    print(f"LiMnO2 2x1x1 on 3x2x2, P = 1/N: imag_self_energy vs 18 pi / h^2 (N2(1) + N2(2)): {worst:.2e}")
    assert worst <= 1e-13


def _loop_gamma(nu, mesh, tets, target, p, temps):
    """[T, 3n] by a plain loop over (cell, tetrahedron, l1, l2, class): each tetrahedron weighted 1 / 6, its corner
    weights times P at that corner and the occupation factor of the class."""
    n1, n2, n3 = mesh
    n_q, nb = nu.shape
    tq = np.array([target // (n2 * n3), (target // n3) % n2, target % n3])
    out = np.zeros((len(temps), nb))
    occ = [lambda x, t=t: 0.0 if t == 0 else 1.0 / np.expm1(H_OVER_KB_K_PER_THZ * x / t) for t in temps]
    for cell in itertools.product(range(n1), range(n2), range(n3)):
        for tet in tets:
            c = (np.array(cell) + tet) % mesh
            qa = (c[:, 0] * n2 + c[:, 1]) * n3 + c[:, 2]
            c2 = (tq - c) % mesh
            qb = (c2[:, 0] * n2 + c2[:, 1]) * n3 + c2[:, 2]
            for l1, l2 in itertools.product(range(nb), repeat=2):
                a, b = nu[qa, l1], nu[qb, l2]
                keep = (a >= CUT) & (b >= CUT)
                for cls, f in enumerate((a + b, b - a, a - b)):
                    order = np.argsort(f, kind="stable")
                    fs = f[order]
                    for l in range(nb):
                        w = nu[target, l]
                        if w < CUT or not (fs[0] <= w < fs[3]):
                            continue
                        wt = tetrahedron_weights(torch.as_tensor(fs)[None], torch.tensor([w]))[2][0].numpy()
                        for i, v in enumerate(order):
                            if not keep[v]:
                                continue
                            pv = p[qa[v], l, l1, l2] / 6.0 * wt[i]
                            for ti, o in enumerate(occ):
                                n_1, n_2 = o(a[v]), o(b[v])
                                fac = 1 + n_1 + n_2 if cls == 0 else (n_1 - n_2 if cls == 1 else -(n_1 - n_2))
                                out[ti, l] += pv * fac
    return out * 18 * math.pi / H_EV_PER_THZ**2


def test_imag_self_energy_against_loop():
    ph, _ = _spring_phonons()
    mesh = (3, 3, 3)
    temps = [0.0, 300.0, 1000.0]
    mesh_t, nu, e, _, tets, _ = ph._three_phonon_mesh(mesh, temps)
    rng = np.random.default_rng(1)
    p = torch.as_tensor(rng.random((27, 3, 3, 3)) * 1e-6)
    t = torch.as_tensor(np.array(temps))
    worst = 0.0
    for target in (1, 5, 13, 26):
        gamma = torch.zeros(len(temps), 3, dtype=f64)
        ph.kernels.imag_self_energy(nu, mesh_t, tets, target, nu[target].contiguous(),
                                    torch.arange(27, dtype=torch.int32), p, t, CUT, gamma)
        want = _loop_gamma(nu.numpy(), mesh_t, tets.numpy(), target, p.numpy(), temps)
        worst = max(worst, np.abs(gamma.numpy() - want).max() / np.abs(want).max())
    print(f"spring crystal 3^3: imag_self_energy spec vs plain loop {worst:.2e}")
    assert worst <= 1e-13


def test_zero_temperature_and_classical_limit(weights030):
    ph = _limno2_spec_ph(weights030)
    mesh = (2, 2, 2)
    q = [0.5, 0.5, 0.0]
    r0 = ph.linewidths(mesh, q, [0.0])
    mesh_t, nu, e, _, tets, _ = ph._three_phonon_mesh(mesh, None)
    target = 6
    p = ph._interaction_strength(mesh, q)
    w = vertex_weights(nu, mesh_t, tets, target, nu[target], torch.arange(8, dtype=torch.int32), CUT).numpy()
    decay = 18 * math.pi / H_EV_PER_THZ**2 * np.einsum("qlab,qlab->l", p, w[..., 0])
    decay = _degenerate_average(torch.as_tensor(decay)[None], nu[target])[0].numpy()
    err0 = np.abs(r0["linewidths"][0] - decay).max() / np.abs(decay).max()
    # classical limit: n -> k T / h nu
    big = [2e5, 4e5]
    r = ph.linewidths(mesh, q, big)
    nu1 = nu.numpy()[:, None, :, None]
    q2 = [((np.array(np.unravel_index(target, mesh)) - np.array(np.unravel_index(i, mesh))) % mesh) for i in range(8)]
    i2 = [np.ravel_multi_index(tuple(c), mesh) for c in q2]
    nu2 = nu.numpy()[i2][:, None, None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        a = np.where(nu1 >= CUT, 1 / nu1, 0.0)
        b = np.where(nu2 >= CUT, 1 / nu2, 0.0)
    cl = np.einsum("qlab,qlab->l", p, (a + b) * w[..., 0] + (a - b) * (w[..., 1] - w[..., 2]))
    cl = 18 * math.pi / H_EV_PER_THZ**2 * KB / H_EV_PER_THZ * cl
    cl = _degenerate_average(torch.as_tensor(cl)[None], nu[target])[0].numpy()
    errs = [np.abs(r["linewidths"][i] / t - cl).max() / np.abs(cl).max() for i, t in enumerate(big)]
    print(f"LiMnO2 2x1x1: T = 0 against the decay term {err0:.2e}; Gamma / T against the classical limit {errs}")
    assert err0 <= 1e-12
    assert errs[1] <= 1e-6 and errs[1] < errs[0]


def test_thermal_conductivity_mode_sum_chunking_and_errors(weights030):
    ph = _limno2_spec_ph(weights030)
    mesh = (2, 2, 2)
    temps = [0.0, 300.0, 1000.0]
    r = ph.thermal_conductivity(mesh, temps)
    k = r["kappa"]
    assert k.shape == (3, 3, 3) and np.all(k[0] == 0)
    assert np.abs(k - k.transpose(0, 2, 1)).max() <= 1e-13 * np.abs(k).max()
    nu, gam, v, c = r["frequencies"], r["linewidths"], r["group_velocities"], r["heat_capacity"]
    vol = abs(np.linalg.det(ph.cell.prim_lattice))
    want = np.zeros((3, 3, 3))
    left = np.zeros(3, dtype=int)
    for ti, t in enumerate(temps):
        for qi, m in itertools.product(range(nu.shape[0]), range(nu.shape[1])):
            if nu[qi, m] < CUT:
                continue
            if gam[ti, qi, m] <= 0:
                left[ti] += 1
                continue
            x = H_OVER_KB_K_PER_THZ * nu[qi, m] / t if t > 0 else np.inf
            cv = KB * x * x * np.exp(x) / np.expm1(x) ** 2 if t > 0 else 0.0
            assert abs(cv - c[ti, qi, m]) <= 1e-14 * KB
            want[ti] += cv * np.outer(v[qi, m], v[qi, m]) / (4 * np.pi * gam[ti, qi, m])
    want *= KAPPA_W_PER_MK / (nu.shape[0] * vol)
    assert np.abs(k - want).max() <= 1e-13 * np.abs(want).max()
    assert list(r["n_zero_linewidth"]) == list(left)
    lw = ph.linewidths(mesh, gamma_mesh(mesh)[3], temps)["linewidths"]
    assert np.abs(lw - gam[:, 3]).max() <= 1e-14 * np.abs(gam).max()
    ph.ph3_chunk_bytes = 1  # one q1 per call
    r1 = ph.thermal_conductivity(mesh, temps)
    err = np.abs(r1["kappa"] - k).max() / np.abs(k).max()
    print(f"LiMnO2 2x1x1, random fc3, 2^3: kappa(300 K) diag {np.diag(k[1])}, chunked vs unchunked {err:.2e}")
    assert err <= 1e-13
    with pytest.raises(ValueError, match="temperatures"):
        ph.thermal_conductivity(mesh, [-1.0])
    with pytest.raises(ValueError, match="temperatures"):
        ph.linewidths(mesh, [0, 0, 0], [float("nan")])
    with pytest.raises(ValueError, match="mesh"):
        ph.linewidths(mesh, [0.25, 0, 0], [300.0])
    no3 = Phonons(ph.force_constants, ph.cell, device="cpu", kernels=ThreePhononSpecKernels())
    for call in (lambda: no3.linewidths(mesh, [0, 0, 0], [300.0]), lambda: no3.thermal_conductivity(mesh, [300.0])):
        with pytest.raises(ValueError, match="third_order=True"):
            call()
    with pytest.raises(ValueError, match="shape"):
        Phonons(ph.force_constants, ph.cell, fc3=np.zeros((1, 2, 3)), device="cpu", kernels=ThreePhononSpecKernels())


def test_chunk_limit_matches_header():
    from chgnet_b200 import _lib

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "chgnet_b200.h")).read(), flags=re.S)
    assert _lib.ISE_MAX_CHUNKS == int(re.search(r"#define CHG_ISE_MAX_CHUNKS\s+(\d+)", src).group(1))
