"""CPU (fp64): group velocities and the linear tetrahedron density of states of chgnet_b200.phonons, with the
specifications of ``chg_dynamical_matrix_derivatives`` and ``chg_tetrahedron_dos`` (oracle/phonons.py).

* single-tetrahedron identities of the closed forms, and a Monte-Carlo histogram;
* a one-atom simple cubic crystal with nearest-neighbour central springs (three independent 1D chains): group
  velocities and the DOS against closed forms, on 3x3x3 and 2x2x2 (two minimum images per neighbour) supercells;
* LiMnO2 2x1x1 with the oracle's compact force constants: group velocities against central differences of the
  frequencies, the sum rules of the (projected) DOS and its independence of the tetrahedra's body diagonal."""
import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import gamma_mesh, tetrahedra
from oracle.phonon_dos import tetrahedron_weights
from oracle.phonons import PhononSpecKernels
from phonon_cells import A, limno2_211_spec, springs


def _vertex_sets():
    rng = np.random.default_rng(11)
    sets = [np.sort(rng.uniform(-1, 2, 4)) for _ in range(20)]
    sets += [np.array(v, dtype=np.float64) for v in ([0, 0, 1, 2], [0, 1, 1, 2], [0, 1, 2, 2], [0, 0, 0, 1],
                                                       [0, 1, 1, 1], [0, 0, 1, 1], [-1, 0.5, 0.5, 0.5])]
    return sets


def _weights(e, w):
    n, g, wt = tetrahedron_weights(torch.as_tensor(e).expand(len(np.atleast_1d(w)), 4), torch.as_tensor(w))
    return n.numpy(), g.numpy(), wt.numpy()


@pytest.mark.parametrize("e", _vertex_sets(), ids=lambda e: ",".join(f"{x:.2f}" for x in e))
def test_single_tetrahedron_identities(e):
    lo, hi = e[0] - 0.1, e[3] + 0.1
    w = np.concatenate([np.linspace(lo, hi, 2001), e])  # the vertices themselves included
    n, g, wt = _weights(e, w)
    scale = 3.0 / max(e[3] - e[0], 1e-300)
    assert np.abs(wt.sum(1) - g).max() <= 1e-13 * scale
    assert np.abs(wt @ e - w * g).max() <= 1e-13 * scale * np.abs(e).max()
    assert (wt >= -1e-15 * scale).all() and (g >= 0).all()
    # n rises monotonically from 0 to 1
    order = np.argsort(w, kind="stable")
    assert n[order][0] == 0 and n[order][-1] == 1 and (np.diff(n[order]) >= -1e-15).all()
    if e[3] == e[0]:
        return
    # int wt_i dw = 1/4: wt is a cubic polynomial between vertices, 3-point Gauss-Legendre is exact
    x, gw = np.polynomial.legendre.leggauss(3)
    total = np.zeros(4)
    for a, b in zip(e[:-1], e[1:]):
        if b > a:
            pts = 0.5 * (b - a) * x + 0.5 * (a + b)
            total += 0.5 * (b - a) * (gw @ _weights(e, pts)[2])
    assert np.abs(total - 0.25).max() <= 1e-13
    # dn/dw = g and dn/de_i = -wt_i by central differences, away from the vertices
    h = 1e-6 * (e[3] - e[0])
    wm = np.linspace(lo, hi, 997)
    wm = wm[np.min(np.abs(wm[:, None] - e[None, :]), axis=1) > 10 * h]
    fd = (_weights(e, wm + h)[0] - _weights(e, wm - h)[0]) / (2 * h)
    assert np.abs(fd - _weights(e, wm)[1]).max() <= 1e-6 * scale
    if len(np.unique(e)) == 4:
        for i in range(4):
            d = np.zeros(4)
            d[i] = h
            fd = (_weights(e + d, wm)[0] - _weights(e - d, wm)[0]) / (2 * h)
            assert np.abs(fd + _weights(e, wm)[2][:, i]).max() <= 1e-6 * scale


def test_single_tetrahedron_monte_carlo():
    rng = np.random.default_rng(5)
    e = np.array([-0.3, 0.4, 0.55, 1.7])
    lam = rng.dirichlet(np.ones(4), size=10**6)  # uniform in the tetrahedron
    eps = lam @ e
    edges = np.linspace(e[0], e[3], 41)
    x, gw = np.polynomial.legendre.leggauss(4)
    n_mc = np.histogram(eps, edges)[0] / len(eps)
    w_mc = np.stack([np.histogram(eps, edges, weights=lam[:, i])[0] / len(eps) for i in range(4)], 1)
    n_edges = _weights(e, edges)[0]
    want_n = np.diff(n_edges)
    want_w = np.zeros((40, 4))
    for b in range(40):  # the bins do not straddle vertices exactly; 4-point Gauss is exact up to degree 7 per piece
        knots = np.unique(np.clip(np.concatenate([edges[b : b + 2], e]), edges[b], edges[b + 1]))
        for a, c in zip(knots[:-1], knots[1:]):
            pts = 0.5 * (c - a) * x + 0.5 * (a + c)
            want_w[b] += 0.5 * (c - a) * (gw @ _weights(e, pts)[2])
    sigma_n = np.sqrt(np.maximum(want_n, 1e-12) / len(eps))
    assert np.abs(n_mc - want_n).max() <= 5 * sigma_n.max()
    assert np.abs(want_w.sum(1) - want_n).max() <= 1e-13
    assert np.abs(w_mc - want_w).max() <= 5 * sigma_n.max()


def _sc_springs(m):
    """One atom per simple cubic cell (lattice constant A), nearest-neighbour central springs: nu_a = nu_max
    |sin pi q_a|."""
    ph, nu_max = springs(m)
    return ph, nu_max[0]


@pytest.mark.parametrize("m", [[3, 3, 3], [2, 2, 2]])
def test_spring_crystal_group_velocities(m):
    ph, nu_max = _sc_springs(m)
    nbr = np.abs(ph.force_constants[0]).sum(axis=(1, 2)) > 0
    nbr[0] = False
    assert (ph.cell.multiplicities[0, nbr] == (2 if m == [2, 2, 2] else 1)).all()  # +-a e_c: one atom, two images
    rng = np.random.default_rng(7)
    q = rng.uniform(-0.5, 0.5, size=(40, 3))
    branch = nu_max * np.abs(np.sin(np.pi * q))  # [Q, 3]: branch a moves along a
    dbranch = nu_max * np.pi * A * np.cos(np.pi * q) * np.sign(np.sin(np.pi * q))  # d nu_a / dQ_a (Q = q / A)
    nu = ph.frequencies(q)
    assert np.abs(nu - np.sort(branch, axis=1)).max() <= 1e-10 * nu_max
    v = ph.group_velocities(q)
    assert v.shape == (40, 3, 3)
    order = np.argsort(branch, axis=1)
    want = np.zeros((40, 3, 3))
    for a in range(3):
        want[np.arange(40)[:, None], np.argsort(order, axis=1)[:, a : a + 1], a] = dbranch[:, a : a + 1]
    vmax = nu_max * np.pi * A
    assert np.abs(v - want).max() <= 1e-10 * vmax
    assert np.abs(ph.group_velocities(q[0]) - v[0]).max() == 0
    # along (t, t, t) the three branches are degenerate: the set's sum is the sum of the branch velocities
    t = np.array([0.13, 0.31, -0.22])
    qd = np.repeat(t[:, None], 3, axis=1)
    vd = ph.group_velocities(qd)
    d = nu_max * np.pi * A * np.cos(np.pi * t) * np.sign(np.sin(np.pi * t))
    assert np.abs(vd.sum(1) - d[:, None]).max() <= 1e-10 * vmax


def test_spring_crystal_dos_converges_to_the_chain():
    ph, nu_max = _sc_springs([3, 3, 3])
    w = np.linspace(0.05, 0.9, 35) * nu_max
    want = 3 * (2 / np.pi) / np.sqrt(nu_max**2 - w**2)
    mean, worst = [], []
    for n in (8, 16, 32):
        out = ph.dos((n, n, n), w)
        rel = np.abs(out["total_dos"] - want) / want.max()
        mean.append(rel.mean())
        worst.append(rel.max())
        assert abs(ph.dos((n, n, n))["integrated_dos"][-1] - 3) <= 1e-12
    print("spring crystal: |dos - 3 (2/pi)/sqrt(nu_max^2 - nu^2)| / max, meshes 8, 16, 32: mean", mean, "max", worst)
    # the error falls as the mesh is refined.  Calibrated on this model (mean 0.069, 0.037, 0.018; max 0.30, 0.13,
    # 0.078): the sorted bands cross all over the zone, and the largest errors sit near 0.9 nu_max where the exact DOS
    # is steep.  The mean is the monotone measure; the maximum is bounded at 32^3.
    assert mean[2] < mean[1] < mean[0] and worst[2] < worst[0]
    assert mean[2] <= 0.025 and worst[2] <= 0.1


@pytest.fixture(scope="module")
def limno2_211_fc(weights030):
    return limno2_211_spec(weights030)


def test_limno2_group_velocities_match_finite_differences(limno2_211_fc):
    ph = limno2_211_fc
    rng = np.random.default_rng(3)
    q = rng.uniform(-0.5, 0.5, size=(8, 3))
    nu = ph.frequencies(q)
    v = ph.group_velocities(q)
    lat = ph.cell.prim_lattice
    h = 1e-6  # 1/A: the difference converges as h^2 (1.1e-4, 1.1e-6, 1.1e-8 at 1e-4, 1e-5, 1e-6)
    fd = np.zeros_like(v)
    for c in range(3):
        dq = h * lat[:, c]  # q = Q lattice^T: a step h along Q_c
        fd[:, :, c] = (ph.frequencies(q + dq) - ph.frequencies(q - dq)) / (2 * h)
    gaps = np.diff(nu, axis=1)
    isolated = np.ones_like(nu, dtype=bool)
    isolated[:, 1:] &= gaps > 1e-2
    isolated[:, :-1] &= gaps > 1e-2
    isolated &= np.abs(nu) > 0.1
    assert isolated.sum() >= 100 and (nu < 0).any()  # imaginary modes included
    err = np.abs(v - fd)[isolated].max() / np.abs(v).max()
    print(f"LiMnO2 2x1x1: max|v - central difference| / max|v| = {err:.2e} over {isolated.sum()} modes")
    assert err <= 1e-7


def test_limno2_dos_sum_rules_and_diagonal(limno2_211_fc):
    ph = limno2_211_fc
    mesh = (6, 5, 4)
    out = ph.dos(mesh, projected=True)
    w, total, pdos = out["frequency_points"], out["total_dos"], out["projected_dos"]
    assert w.shape == (201,) and pdos.shape == (8, 201)
    assert abs(out["integrated_dos"][-1] - 24) <= 1e-12 and out["integrated_dos"][0] <= 1e-12
    assert np.abs(pdos.sum(0) - total).max() <= 1e-12 * total.max()
    assert (np.diff(out["integrated_dos"]) >= -1e-12).all()
    # the body diagonal of the tetrahedra changes the result only by the discretisation
    nu = torch.as_tensor(ph.frequencies(gamma_mesh(mesh)))
    kern = PhononSpecKernels()
    dos = []
    for d in range(4):
        tot, idos = torch.empty(201, dtype=torch.float64), torch.empty(201, dtype=torch.float64)
        kern.tetrahedron_dos(nu, mesh, torch.as_tensor(tetrahedra(mesh, ph.cell.prim_lattice, d)), torch.as_tensor(w),
                             tot, idos)
        assert abs(float(idos[-1]) - 24) <= 1e-12
        dos.append(tot.numpy())
    chosen = tetrahedra(mesh, ph.cell.prim_lattice)
    assert any((chosen == tetrahedra(mesh, ph.cell.prim_lattice, d)).all() for d in range(4))
    # LiMnO2 is orthorhombic with mirror planes normal to the axes: the reflected decompositions are mirror images
    # of each other on its bands, so the four agree to rounding
    spread = max(np.abs(a - dos[0]).max() for a in dos[1:]) / dos[0].max()
    print(f"LiMnO2 2x1x1, mesh {mesh}: max over diagonals of |dos_d - dos_0| / max = {spread:.2e}")
    assert spread <= 1e-12


def test_tetrahedron_diagonals_agree_within_discretisation():
    """A band with no mirror symmetry: the four diagonals give different tetrahedra and agree to the discretisation
    error, which falls with the mesh."""
    lat = graphgen.limno2_structure()[2]
    kern = PhononSpecKernels()
    w = torch.linspace(-1.2, 1.2, 49, dtype=torch.float64)
    spreads = []
    for n in (12, 24):
        q = gamma_mesh((n, n, n))
        band = np.cos(2 * np.pi * (q[:, 0] + 0.3 * q[:, 1])) + 0.4 * np.sin(2 * np.pi * (q[:, 1] - q[:, 2]))
        nu = torch.as_tensor(band[:, None])
        idos = []
        for d in range(4):
            tot, i = torch.empty(49, dtype=torch.float64), torch.empty(49, dtype=torch.float64)
            kern.tetrahedron_dos(nu, (n, n, n), torch.as_tensor(tetrahedra((n, n, n), lat, d)), w, tot, i)
            idos.append(i.numpy())
        spreads.append(max(np.abs(a - idos[0]).max() for a in idos[1:]))
    print("skewed band: max over diagonals of |idos_d - idos_0|, meshes 12, 24:", spreads)
    assert 0 < spreads[1] < spreads[0] <= 1e-2
