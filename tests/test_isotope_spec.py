"""CPU (fp64): isotope and boundary scattering of chgnet_b200.phonons with the specification of
``chg_isotope_scattering`` (tests/isotope_kernels.py), DESIGN.md section 12.11.

* completeness: summed over the target's bands at one frequency, Gamma^iso is (pi / 4) w^2 sum_k g_k pdos_k(w), on
  LiMnO2 2x1x1 and on random unitary eigenvectors (a sum over a complete basis at the target, so neither planted bug
  can move it);
* a plain loop over the vertices q' and their 24 (tetrahedron, corner) with ``np.vdot`` overlaps; both planted bugs
  miss it;
* rotating the crystal rigidly leaves the degenerate-averaged ``isotope_linewidths`` unchanged, and the
  per-component bug does not;
* on a 1D spring chain Gamma^iso approaches Tamura's rate with the exact 1D density of states;
* Gamma^iso is linear in g and 0 for g = 0;
* boundary scattering alone gives the closed-form kappa, proportional to L, and kappa_LBTE = kappa_RTA with S = 0;
* wiring of the three conductivities, chunking, the header limit and the input errors."""
import os
import re

import numpy as np
import pytest
import torch

from chgnet_b200 import _lib
from chgnet_b200.phonons import KAPPA_W_PER_MK, THERMAL_CUTOFF_THZ, Phonons, gamma_mesh, make_supercell, tetrahedra
from isotope_kernels import IsotopeSpecKernels
from oracle.phonons import PhononSpecKernels
from phonon_cells import limno2_211, springs
from test_three_phonon_spec import KS, _random_symmetric_fc3

CUT = THERMAL_CUTOFF_THZ
TEMPS = [0.0, 300.0, 1000.0]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# illustrative mass variances of LiMnO2's 8 primitive atoms (2 Li, 2 Mn, 4 O); not natural-abundance data
G_LIMNO2 = [1.5e-3, 1.5e-3, 0.0, 0.0, 3.4e-5, 3.4e-5, 3.4e-5, 3.4e-5]


@pytest.fixture(scope="module")
def limno2(weights030):
    sc, _, fc = limno2_211(weights030)
    return fc, sc, _random_symmetric_fc3(sc, 3)[1]


def _ph(fc, sc, fc3=None, **kw):
    return Phonons(fc, sc, fc3=fc3, device="cpu", kernels=IsotopeSpecKernels(**kw))


def _completeness(nu, e, mesh, tets, g, targets, w0s, kernels):
    """max over w0 and the targets of |sum_l Gamma_l(w0) - (pi / 4) w0^2 sum_k g_k pdos_k(w0)| / that value."""
    n_q, nb = nu.shape
    n_prim = nb // 3
    proj = (e.abs() ** 2).view(n_q, nb, n_prim, 3).sum(-1)  # mode-major: [q, mode, atom]
    proj = torch.where((nu >= CUT)[..., None], proj, 0.0)
    omega = torch.as_tensor(w0s, dtype=torch.float64)
    dos, idos, pdos = torch.empty_like(omega), torch.empty_like(omega), torch.empty(n_prim, len(w0s), dtype=torch.float64)
    PhononSpecKernels().tetrahedron_dos(nu, mesh, tets, omega, dos, idos, proj, pdos)
    worst = 0.0
    for i, w0 in enumerate(w0s):
        om = torch.full((len(targets), nb), float(w0), dtype=torch.float64)
        gamma = torch.empty_like(om)
        kernels.isotope_scattering(nu, mesh, tets, e, g, torch.as_tensor(targets, dtype=torch.int32), om, CUT, gamma)
        want = np.pi / 4 * w0**2 * float((g * pdos[:, i]).sum())
        assert want > 0
        worst = max(worst, float((gamma.sum(1) - want).abs().max()) / want)
    return worst


def test_completeness_limno2(limno2):
    fc, sc, _ = limno2
    ph = _ph(fc, sc)
    mesh, nu, e, _, tets = ph._mesh_modes((3, 2, 2))
    g = torch.as_tensor(G_LIMNO2, dtype=torch.float64)
    w0s = [float(nu[4, 5]) + 1e-3, float(nu[7, 12]) + 1e-3, float(nu[2, 20]) + 1e-3]  # inside bands, not in a gap
    targets = [1, 5, 11]
    err = _completeness(nu, e, mesh, tets, g, targets, w0s, IsotopeSpecKernels())
    print(f"LiMnO2 2x1x1 on 3x2x2: sum_l Gamma_l(w0) vs (pi/4) w0^2 sum g pdos {err:.2e}")
    assert err <= 1e-13


def test_completeness_random_unitary():
    gen = torch.Generator().manual_seed(7)
    mesh, nb = (4, 3, 2), 12
    n_q = 24
    nu = torch.sort(torch.rand(n_q, nb, generator=gen, dtype=torch.float64) * 12.0 - 1.0, dim=1)[0]
    nu[:, 0] = 5e-4  # below the cutoff
    a = torch.complex(torch.randn(n_q, nb, nb, generator=gen, dtype=torch.float64),
                      torch.randn(n_q, nb, nb, generator=gen, dtype=torch.float64))
    e = torch.linalg.qr(a)[0].mT.contiguous()
    g = torch.rand(nb // 3, generator=gen, dtype=torch.float64) * 1e-3
    tets = torch.as_tensor(tetrahedra(mesh, np.eye(3)))
    w0s = [1.5, 4.0, 7.3, 10.0]
    err = _completeness(nu, e, mesh, tets, g, [0, 7, 23], w0s, IsotopeSpecKernels())
    print(f"random unitary eigenvectors, 12 bands on 4x3x2: completeness {err:.2e}")
    assert err <= 1e-13


def _loop_gamma(nu, e, mesh, tets, g, target, omega):
    """Gamma [nb] by plain loops: (pi / 4) w^2 (1/N) sum over q' and l' of W O, W = 1/6 of the weights of corner q' in
    the 24 (tetrahedron, corner) that have it, O = sum_k g_k |vdot(e_k(target, l), e_k(q', l'))|^2."""
    from oracle.phonon_dos import tetrahedron_weights

    n1, n2, n3 = mesh
    nu, e, off = nu.numpy(), e.numpy(), tets.numpy()
    n_q, nb = nu.shape
    out = np.zeros(nb)
    for qp in range(n_q):
        c = np.array([qp // (n2 * n3), (qp // n3) % n2, qp % n3])
        for lp in range(nb):
            if nu[qp, lp] < CUT:
                continue
            for it in range(6):
                for v in range(4):
                    cell = c - off[it, v]
                    qs = [int(np.ravel_multi_index(tuple((cell + off[it, u]) % mesh), mesh)) for u in range(4)]
                    ev = nu[qs, lp]
                    order = np.argsort(ev, kind="stable")
                    for l in range(nb):
                        if omega[l] < CUT:
                            continue
                        wt = tetrahedron_weights(torch.as_tensor(ev[order]), float(omega[l]))[2].numpy()
                        o = sum(g[k] * abs(np.vdot(e[target, l, 3 * k : 3 * k + 3], e[qp, lp, 3 * k : 3 * k + 3])) ** 2
                                for k in range(nb // 3))
                        out[l] += wt[list(order).index(v)] / 6.0 * o
    return np.pi / 4 * omega**2 * out / n_q


def test_plain_loop():
    gen = torch.Generator().manual_seed(5)
    mesh, nb = (3, 2, 2), 6
    n_q = 12
    nu = torch.sort(torch.rand(n_q, nb, generator=gen, dtype=torch.float64) * 6.0 - 0.5, dim=1)[0]
    nu[::4, 0] = 5e-4
    a = torch.complex(torch.randn(n_q, nb, nb, generator=gen, dtype=torch.float64),
                      torch.randn(n_q, nb, nb, generator=gen, dtype=torch.float64))
    e = torch.linalg.qr(a)[0].mT.contiguous()
    g = torch.tensor([1.1e-3, 4.0e-4], dtype=torch.float64)
    tets = torch.as_tensor(tetrahedra(mesh, np.eye(3), diagonal=2))
    targets = torch.tensor([0, 5, 11], dtype=torch.int32)
    omega = torch.rand(3, nb, generator=gen, dtype=torch.float64) * 5.0
    omega[1, 2] = 5e-4
    want = np.stack([_loop_gamma(nu, e, mesh, tets, g.numpy(), int(t), omega[i].numpy()) for i, t in enumerate(targets)])
    errs = {}
    for name, kw in (("spec", {}), ("conj", {"conj_target": False}), ("component", {"per_component": True})):
        got = torch.empty(3, nb, dtype=torch.float64)
        IsotopeSpecKernels(**kw).isotope_scattering(nu, mesh, tets, e, g, targets, omega, CUT, got)
        errs[name] = float(np.abs(got.numpy() - want).max() / np.abs(want).max())
    print(f"random unitary eigenvectors, 6 bands on 3x2x2: specification vs plain loop {errs['spec']:.2e}; unconjugated "
          f"target {errs['conj']:.2e}; per-component {errs['component']:.2e}")
    assert want[1, 2] == 0 and np.abs(want).max() > 0
    assert errs["spec"] <= 1e-14 and errs["conj"] > 1e-3 and errs["component"] > 1e-3


def test_rotation_invariance(limno2):
    fc, sc, _ = limno2
    r = np.linalg.qr(np.random.default_rng(3).standard_normal((3, 3)))[0]
    sc_r = make_supercell(sc.prim_z, sc.prim_frac, sc.prim_lattice @ r.T, [2, 1, 1])
    fc_r = np.einsum("ab,kjbc,dc->kjad", r, fc, r)
    mesh = (3, 2, 2)
    q = gamma_mesh(mesh)
    out = {}
    for name, kw in (("spec", {}), ("bug", {"per_component": True})):
        base = _ph(fc, sc, **kw).isotope_linewidths(mesh, q, G_LIMNO2)
        rot = _ph(fc_r, sc_r, **kw).isotope_linewidths(mesh, q, G_LIMNO2)
        top = np.abs(base["isotope_linewidths"]).max()
        out[name] = np.abs(rot["isotope_linewidths"] - base["isotope_linewidths"]).max() / top
    print(f"LiMnO2 2x1x1 on 3x2x2 rotated rigidly: isotope_linewidths change {out['spec']:.2e} of max; per-component "
          f"bug {out['bug']:.2e}")
    # the rotated eigensolve splits near-degenerate sets differently by ~1e-12 of the largest value (measured 2.3e-12)
    assert out["spec"] <= 1e-11 and out["bug"] > 1e-3


@pytest.mark.parametrize("n", [64, 256])
def test_continuum_limit(n):
    ph, nu_max = springs((1, 1, 3))
    vmax = nu_max[2]
    g = 2.0e-3
    mesh = (1, 1, n)
    res = ph.__class__(ph.force_constants, ph.cell, device="cpu", kernels=IsotopeSpecKernels()).isotope_linewidths(
        mesh, gamma_mesh(mesh), [g])
    nu, gam = res["frequencies"][:, 2], res["isotope_linewidths"][:, 2]
    sel = (nu >= 0.25 * vmax) & (nu <= 0.75 * vmax)
    want = g * nu[sel] ** 2 / (2 * np.sqrt(vmax**2 - nu[sel] ** 2))
    err = float(np.abs(gam[sel] / want - 1).max())
    print(f"spring chain on 1x1x{n}: {int(sel.sum())} targets in [0.25, 0.75] nu_max, Gamma^iso vs g nu^2 / "
          f"(2 sqrt(nu_max^2 - nu^2)) {err:.2e}; other branches {np.abs(res['isotope_linewidths'][:, :2]).max():.1e}")
    assert np.all(res["isotope_linewidths"][:, :2] == 0)
    # the O(1/n) chord error of the linear interpolation: measured 7.0e-3 on 1x1x256 and 2.8e-2 on 1x1x64
    assert err <= (1e-2 if n == 256 else 4e-2)


def test_scalings(limno2):
    fc, sc, _ = limno2
    ph = _ph(fc, sc)
    mesh = (2, 2, 2)
    q = gamma_mesh(mesh)
    g = np.asarray(G_LIMNO2)
    base = ph.isotope_linewidths(mesh, q, g)["isotope_linewidths"]
    assert np.abs(base).max() > 0
    assert np.array_equal(ph.isotope_linewidths(mesh, q, 4.0 * g)["isotope_linewidths"], 4.0 * base)
    three = ph.isotope_linewidths(mesh, q, 3.0 * g)["isotope_linewidths"]
    assert np.abs(three - 3.0 * base).max() <= 1e-15 * np.abs(base).max()
    assert np.all(ph.isotope_linewidths(mesh, q, np.zeros(8))["isotope_linewidths"] == 0)
    one = ph.isotope_linewidths(mesh, q[3], g)
    assert one["isotope_linewidths"].shape == (24,) and np.array_equal(one["isotope_linewidths"], base[3])
    assert np.all(base[0, :3] == 0)  # the Gamma acoustic modes


def _boundary_closed_form(res, l_um, vol):
    v = res["group_velocities"]
    speed = np.linalg.norm(v, axis=-1)
    vhat = np.where(speed[..., None] > 0, v / np.where(speed > 0, speed, 1.0)[..., None], 0.0)
    n_q = v.shape[0]
    return (1e4 * l_um / (n_q * vol) * KAPPA_W_PER_MK
            * np.einsum("tqm,qm,qma,qmb->tab", res["heat_capacity"], speed, vhat, vhat))


def test_boundary_only():
    ph0, _ = springs((3, 3, 3), ks=KS)
    sc = ph0.cell
    fc3 = np.zeros((1, len(sc.z), len(sc.z), 3, 3, 3))
    ph = _ph(ph0.force_constants, sc, fc3)
    mesh = (3, 3, 3)
    vol = abs(np.linalg.det(sc.prim_lattice))
    res = ph.thermal_conductivity(mesh, TEMPS, boundary_mfp=0.5)
    res2 = ph.thermal_conductivity(mesh, TEMPS, boundary_mfp=1.0)
    want = _boundary_closed_form(res, 0.5, vol)
    top = np.abs(want).max()
    err = np.abs(res["kappa"] - want).max() / top
    lin = np.abs(res2["kappa"] - 2.0 * res["kappa"]).max() / top
    lbte = ph.thermal_conductivity_lbte(mesh, TEMPS, boundary_mfp=0.5)
    s = ph._collision_matrix(mesh, TEMPS)[0]
    err_lbte = np.abs(lbte["kappa"] - res["kappa"]).max() / top
    print(f"spring crystal ks {KS}, fc3 = 0, L = 0.5 um on 3^3: kappa vs closed form {err:.2e}, kappa(2L) vs 2 kappa(L) "
          f"{lin:.2e}, kappa_LBTE vs kappa_RTA {err_lbte:.2e}; 300 K diagonal {np.diag(res['kappa'][1])} W/(m K)")
    assert top > 0 and np.all(res["linewidths"] == 0) and np.all(res["kappa"][0] == 0)
    assert err <= 1e-13 and lin <= 1e-13
    assert torch.all(s == 0) and np.array_equal(lbte["kappa_rta"], res["kappa"]) and err_lbte <= 1e-12
    assert "isotope_linewidths" not in res and res["boundary_linewidths"].shape == res["frequencies"].shape


def test_wiring(limno2):
    fc, sc, fc3 = limno2
    ph = _ph(fc, sc, fc3)
    mesh = (2, 2, 2)
    opts = {"mass_variances": G_LIMNO2, "boundary_mfp": 0.2}
    plain = ph.thermal_conductivity(mesh, TEMPS)
    zero = ph.thermal_conductivity(mesh, TEMPS, mass_variances=np.zeros(8))
    assert np.array_equal(zero["kappa"], plain["kappa"]) and np.array_equal(zero["linewidths"], plain["linewidths"])
    assert np.all(zero["isotope_linewidths"] == 0)
    rta = ph.thermal_conductivity(mesh, TEMPS, **opts)
    lbte = ph.thermal_conductivity_lbte(mesh, TEMPS, **opts)
    wig = ph.thermal_conductivity_wigner(mesh, TEMPS, **opts)
    assert np.array_equal(rta["linewidths"], plain["linewidths"])
    assert np.array_equal(lbte["kappa_rta"], rta["kappa"]) and np.array_equal(wig["kappa_p"], rta["kappa"])
    assert np.array_equal(wig["kappa"], wig["kappa_p"] + wig["kappa_c"])
    for res in (lbte, wig):
        assert np.array_equal(res["isotope_linewidths"], rta["isotope_linewidths"])
        assert np.array_equal(res["boundary_linewidths"], rta["boundary_linewidths"])
    iso = ph.isotope_linewidths(mesh, gamma_mesh(mesh), G_LIMNO2)["isotope_linewidths"]
    assert np.array_equal(rta["isotope_linewidths"], iso)
    drop = np.diag(rta["kappa"][1]) / np.diag(plain["kappa"][1])
    print(f"LiMnO2 2x1x1 on 2^3 at 300 K: kappa with isotopes and L = 0.2 um over kappa without {drop}; LBTE "
          f"{np.diag(lbte['kappa'][1])}, Wigner {np.diag(wig['kappa'][1])} W/(m K)")
    assert np.all(drop < 1) and np.all(drop > 0)
    assert np.array_equal(lbte["n_zero_linewidth"], rta["n_zero_linewidth"])


def test_chunking_header_and_errors(limno2):
    fc, sc, fc3 = limno2
    ph = _ph(fc, sc, fc3)
    mesh = (2, 2, 2)
    q = gamma_mesh(mesh)
    base = ph.isotope_linewidths(mesh, q, G_LIMNO2)
    ph.isotope_chunk_bytes = 1  # one target per call
    assert np.array_equal(ph.isotope_linewidths(mesh, q, G_LIMNO2)["isotope_linewidths"], base["isotope_linewidths"])
    ph.isotope_chunk_bytes = Phonons.isotope_chunk_bytes
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "chgnet_b200.h")).read(), flags=re.S)
    assert _lib.ISO_MAX_CHUNKS == int(re.search(r"#define CHG_ISO_MAX_CHUNKS\s+(\d+)", src).group(1))
    assert _lib.isotope_scratch_doubles(5, 7, 6) == 5 * 7 * 36 + _lib.ISO_MAX_CHUNKS * 5 * 6
    no3 = _ph(fc, sc)
    assert np.array_equal(no3.isotope_linewidths(mesh, q, G_LIMNO2)["isotope_linewidths"], base["isotope_linewidths"])
    with pytest.raises(ValueError, match="third_order=True"):
        no3.thermal_conductivity(mesh, [300.0], mass_variances=G_LIMNO2)
    bad_g = [G_LIMNO2[:7], G_LIMNO2 + [0.0], [-1e-4] + G_LIMNO2[1:], [float("nan")] + G_LIMNO2[1:],
             [float("inf")] + G_LIMNO2[1:]]
    for g in bad_g:
        with pytest.raises(ValueError, match="mass_variances"):
            ph.isotope_linewidths(mesh, q, g)
    with pytest.raises(ValueError, match="mesh"):
        ph.isotope_linewidths(mesh, [0.25, 0.0, 0.0], G_LIMNO2)
    methods = (ph.thermal_conductivity, ph.thermal_conductivity_lbte, ph.thermal_conductivity_wigner)
    for method in methods:
        for g in bad_g:
            with pytest.raises(ValueError, match="mass_variances"):
                method(mesh, [300.0], mass_variances=g)
        for mfp in (0.0, -1.0, float("nan"), float("inf")):
            with pytest.raises(ValueError, match="boundary_mfp"):
                method(mesh, [300.0], boundary_mfp=mfp)
        with pytest.raises(ValueError, match="temperatures"):
            method(mesh, [-1.0], mass_variances=G_LIMNO2)
