"""CPU (fp64): the velocity operator and the Wigner coherence conductivity of chgnet_b200.phonons with the specification
of ``chg_coherence_conductivity`` (tests/wigner_kernels.py), DESIGN.md section 12.10.

* V: Hermitian; its diagonal is ``group_velocities`` for non-degenerate modes; its squared norm over a degenerate set
  is the set's sum of squared group velocities; it equals the central differences of ``dynamical_matrices`` sandwiched
  between the eigenvectors (the phase convention);
* the pair sum restricted to s = s' is kappa_RTA, and restricted to the same-set pairs its diagonal is kappa_RTA's;
* kappa_C does not depend on the basis inside degenerate sets, and the same-set bug does;
* on the spring crystal with cubic chain terms kappa_C is 0 (V vanishes between polarisations);
* fc3 scaling, the weak-coupling limit, symmetry and T = 0;
* chunking, one temperature, kappa_p bitwise ``thermal_conductivity``'s kappa, input errors and the header limit."""
import os
import re

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.phonons import (KAPPA_W_PER_MK, THERMAL_CUTOFF_THZ, THZ_PER_SQRT_EV_A2_AMU, Phonons,
                                 _degenerate_set_ids, make_supercell)
from oracle.phonons import oracle_compact_fcs
from phonon_cells import CU, K, limno2_211, springs
from test_three_phonon_spec import KS, _chain_fc3, _random_symmetric_fc3
from three_phonon_kernels import ThreePhononSpecKernels
from wigner_kernels import WignerSpecKernels, coherence_sum, rotate_sets, velocity_operator

CUT = THERMAL_CUTOFF_THZ
TEMPS = [0.0, 300.0, 1000.0]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Recording(WignerSpecKernels):
    """Records the arguments of every ``coherence_conductivity`` call."""

    def __init__(self):
        super().__init__()
        self.calls = []

    def coherence_conductivity(self, freqs, eigvecs, ddyn, set_id, heat_capacity, gamma, cutoff_thz, kappa):
        self.calls.append((freqs.clone(), eigvecs.clone(), ddyn.clone(), set_id.clone(), heat_capacity.clone(),
                           gamma.clone()))
        super().coherence_conductivity(freqs, eigvecs, ddyn, set_id, heat_capacity, gamma, cutoff_thz, kappa)


def _run(fc, sc, fc3, mesh, temps=TEMPS):
    """(thermal_conductivity_wigner's result on the spec path, its kernel inputs concatenated over the calls, the scale
    KAPPA_W_PER_MK / (N V0))."""
    rec = _Recording()
    ph = Phonons(fc, sc, fc3=fc3, device="cpu", kernels=rec)
    res = ph.thermal_conductivity_wigner(mesh, temps)
    nu, e, dd, sid = (torch.cat([c[i] for c in rec.calls]) for i in range(4))
    cv, g = (torch.cat([c[i] for c in rec.calls], 1) for i in (4, 5))
    scale = KAPPA_W_PER_MK / (nu.shape[0] * abs(np.linalg.det(sc.prim_lattice)))
    return res, (nu, e, dd, sid, cv, g), scale


def _kappa_c(inputs, scale, kernels):
    nu, e, dd, sid, cv, g = inputs
    k = torch.zeros(cv.shape[0], 3, 3, dtype=torch.float64)
    kernels.coherence_conductivity(nu, e, dd, sid, cv, g, CUT, k)
    return k.numpy() * scale


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max())


@pytest.fixture(scope="module")
def limno2(weights030):
    sc, _, fc = limno2_211(weights030)
    return fc, sc, _random_symmetric_fc3(sc, 3)[1]


@pytest.fixture(scope="module")
def cu(weights030):
    sc = make_supercell(*CU, [2, 2, 2])
    g = graphgen.make_crystal_graph(sc.z, sc.frac, sc.lattice)
    return oracle_compact_fcs(weights030, g, sc.p2s), sc, _random_symmetric_fc3(sc, 5)[1]


def _chain(ks):
    ph, _ = springs((3, 3, 3), ks=ks)
    return ph.force_constants, ph.cell, _chain_fc3(ph.cell)


def _velocities(fc, sc, q):
    """(nu [Q, nb], mode-major e, V [Q, 3, nb, nb], group_velocities [Q, nb, 3], the Phonons) at the reduced q."""
    ph = Phonons(fc, sc, device="cpu", kernels=ThreePhononSpecKernels())
    nu, vecs = ph.frequencies(q, eigenvectors=True)
    nu, e = torch.as_tensor(nu), torch.as_tensor(vecs).mT.contiguous()
    nb = nu.shape[1]
    dd = torch.empty(len(q), 3, nb, nb, dtype=torch.complex128)
    ph.kernels.dynamical_matrix_derivatives(ph._fc, ph._img_ptr, ph._img_vec, ph._s2p, ph._inv_sqrt_m,
                                            torch.as_tensor(q), ph._lattice, dd)
    return nu, e, velocity_operator(nu, e, dd), ph.group_velocities(q), ph


Q_OFF = np.array([[0.13, 0.27, 0.41], [0.31, -0.17, 0.09], [0.45, 0.05, 0.22]])
Q_CU = np.array([[0.25, 0.25, 0.25], [0.5, 0.5, 0.5], [0.1, 0.1, 0.1], [0.25, 0.0, 0.25], [0.13, 0.27, 0.41]])


@pytest.mark.parametrize("cell", ["limno2", "cu"])
def test_velocity_operator_diagonal_and_sets(cell, limno2, cu):
    fc, sc, _ = limno2 if cell == "limno2" else cu
    q = np.concatenate([Q_OFF, np.array([[0.5, 0.0, 0.0], [0.0, 0.5, 0.5], [0.5, 0.5, 0.5]])]) if cell == "limno2" \
        else Q_CU
    nu, _, v, gv, _ = _velocities(fc, sc, q)
    herm = float((v - v.mH).abs().max() / v.abs().max())
    sid = _degenerate_set_ids(nu)
    diag = sets = 0.0
    n_sets = 0
    for i in range(len(q)):
        for s in torch.unique(sid[i]):
            idx = torch.nonzero((sid[i] == s) & (nu[i] >= CUT))[:, 0]
            if len(idx) == 0:
                continue
            if len(idx) == 1:
                diag = max(diag, float((v[i, :, idx[0], idx[0]].real - torch.as_tensor(gv[i, idx[0]])).abs().max()))
                continue
            n_sets += 1
            block = (v[i][:, idx][:, :, idx].abs() ** 2).sum((1, 2))
            want = torch.as_tensor((gv[i, idx.numpy()] ** 2).sum(0))
            sets = max(sets, float((block - want).abs().max()))
    scale = float(np.abs(gv).max())
    sets /= scale**2
    print(f"{cell}: V Hermitian to {herm:.2e} of max|V|; diagonal vs group_velocities {diag / scale:.2e} of max|v|; "
          f"{n_sets} degenerate sets, sum |V|^2 vs sum v^2 {sets:.2e} of max v^2")
    assert herm <= 1e-15 and diag <= 1e-14 * scale
    assert sets <= 1e-10  # measured 3.0e-11
    assert cell == "cu" or n_sets > 0  # this Cu's degenerate sets are imaginary modes


def test_velocity_operator_central_differences(limno2):
    fc, sc, _ = limno2
    nu, e, v, _, ph = _velocities(fc, sc, Q_OFF)
    h = 1e-5
    a = torch.as_tensor(nu).abs()
    den = a[:, :, None] + a[:, None, :]
    worst = 0.0
    for c in range(3):
        step = h * sc.prim_lattice[:, c]  # dq_i / dQ_c = lattice[i, c]
        d = (ph.dynamical_matrices(Q_OFF + step) - ph.dynamical_matrices(Q_OFF - step)) / (2 * h)
        fd = THZ_PER_SQRT_EV_A2_AMU**2 * (e.conj() @ d @ e.mT) / den
        worst = max(worst, float((fd - v[:, c]).abs().max() / v.abs().max()))
    print(f"LiMnO2 2x1x1 at 3 off-symmetry q: V vs central differences of D (h = {h}) {worst:.2e} of max|V|")
    assert worst <= 1e-8  # measured 3.5e-9


@pytest.fixture(scope="module")
def limno2_333(limno2):
    return _run(*limno2, (3, 3, 3))


def test_reduction_to_rta(limno2, limno2_333):
    res, (nu, e, dd, sid, cv, g), scale = limno2_333
    v = velocity_operator(nu, e, dd)
    keep = (nu >= CUT)[None] & (g > 0)
    eye = torch.eye(nu.shape[1], dtype=torch.bool)
    diag = coherence_sum(nu, v, cv, g, keep[..., :, None] & keep[..., None, :] & eye).numpy() * scale
    err = _rel(diag, res["kappa_p"])
    res2, (nu, e, dd, sid, cv, g), scale = _run(*limno2, (2, 2, 2))
    v = velocity_operator(nu, e, dd)
    keep = (nu >= CUT)[None] & (g > 0)
    same = keep[..., :, None] & keep[..., None, :] & (sid[:, :, None] == sid[:, None, :])[None]
    n_multi = int(((sid[:, :, None] == sid[:, None, :]) & ~eye).sum())
    block = coherence_sum(nu, v, cv, g, same).numpy() * scale
    err_set = _rel(np.diagonal(block, axis1=1, axis2=2), np.diagonal(res2["kappa_p"], axis1=1, axis2=2))
    print(f"LiMnO2 2x1x1: s = s' pairs vs kappa_RTA on 3^3 (no degenerate kept modes) {err:.2e}; same-set pairs vs "
          f"kappa_RTA diagonal on 2^3 ({n_multi} off-diagonal same-set pairs) {err_set:.2e}")
    # the sets of this cell are split by up to ~1e-6 THz (force-constant noise): the same-set identity holds to that
    assert err <= 1e-14 and n_multi > 0 and err_set <= 2e-8  # measured 1.9e-16 and 5.3e-9


# LiMnO2 2x1x1 on 2^3 has degenerate sets at the zone boundary; the equal-spring crystal has sets across polarisations
@pytest.mark.parametrize("cell", ["limno2", "springs"])
def test_basis_invariance(cell, limno2):
    fc, sc, fc3 = limno2 if cell == "limno2" else _chain((K, K, K))
    mesh = (2, 2, 2) if cell == "limno2" else (3, 3, 3)
    res, inputs, scale = _run(fc, sc, fc3, mesh)
    base = _kappa_c(inputs, scale, WignerSpecKernels())
    rot = _kappa_c(inputs, scale, WignerSpecKernels(rotation_seed=11))
    bug = _kappa_c(inputs, scale, WignerSpecKernels(same_set_pairs=True))
    bug_rot = _kappa_c(inputs, scale, WignerSpecKernels(same_set_pairs=True, rotation_seed=11))
    top = max(np.abs(base).max(), np.abs(res["kappa_p"]).max())
    err = float(np.abs(rot - base).max() / top)
    moved = float(np.abs(bug_rot - bug).max() / top)
    print(f"{cell} on {mesh}: kappa_C with eigenvectors rotated inside degenerate sets {err:.2e} of max(|kappa_C|, "
          f"|kappa_P|) ({np.abs(base).max():.3e}); the same-set bug moves by {moved:.2e} of it")
    assert np.array_equal(res["kappa_c"], base)
    # exact degeneracies (springs) give rounding; LiMnO2's sets are split by up to ~1e-6 THz, and its invariance holds
    # to that spread (measured 1.5e-7)
    assert err <= (1e-12 if cell == "springs" else 1e-6) and moved > 1e-1


@pytest.mark.parametrize("ks", [KS, (K, K, K)])
def test_spring_crystal_kappa_c_vanishes(ks):
    res, inputs, scale = _run(*_chain(ks), (3, 3, 3))
    rot = _kappa_c(inputs, scale, WignerSpecKernels(rotation_seed=5))
    bug = _kappa_c(inputs, scale, WignerSpecKernels(same_set_pairs=True, rotation_seed=5))
    top = np.abs(res["kappa_p"]).max()
    print(f"spring crystal ks {ks}: max|kappa_C| {np.abs(res['kappa_c']).max():.2e}, rotated {np.abs(rot).max():.2e}, "
          f"same-set bug rotated {np.abs(bug).max():.2e}, max|kappa_P| {top:.3e} W/(m K)")
    assert top > 0
    assert np.abs(res["kappa_c"]).max() <= 1e-14 * top and np.abs(rot).max() <= 1e-14 * top
    if ks == (K, K, K):
        assert np.abs(bug).max() > 1e-3 * top


def test_limits(limno2, limno2_333):
    fc, sc, fc3 = limno2
    res, inputs, scale = limno2_333
    res2 = _run(fc, sc, 2.0 * fc3, (3, 3, 3))[0]
    assert np.array_equal(res2["linewidths"], 4.0 * res["linewidths"])
    assert np.array_equal(res2["kappa_p"], res["kappa_p"] / 4.0)
    nu, e, dd, sid, cv, g = inputs
    ratios = []
    for a in (1e-2, 1e-3):
        ratios.append(_kappa_c((nu, e, dd, sid, cv, a * a * g), scale, WignerSpecKernels())[1:] / (a * a))
    r = ratios[0] / res["kappa_c"][1:]
    conv = _rel(ratios[0], ratios[1])
    diag = np.diagonal(r, axis1=1, axis2=2)
    print(f"LiMnO2 2x1x1 on 3^3: fc3 x 2 gives Gamma x 4 and kappa_P / 4 bitwise; kappa_C(a) / a^2 at a = 1e-2 vs "
          f"1e-3 {conv:.2e}; its ratio to kappa_C(1) diagonal {diag.tolist()}")
    assert conv <= 4e-3  # measured 2.0e-3
    assert np.array_equal(res["kappa_c"], res["kappa_c"].transpose(0, 2, 1))
    assert np.all(res["kappa_c"][0] == 0)
    assert np.array_equal(res["kappa"], res["kappa_p"] + res["kappa_c"])


def test_plumbing(limno2):
    fc, sc, fc3 = limno2
    mesh = (2, 2, 2)
    ph = Phonons(fc, sc, fc3=fc3, device="cpu", kernels=WignerSpecKernels())
    base = ph.thermal_conductivity_wigner(mesh, TEMPS)
    assert np.array_equal(base["kappa_p"], ph.thermal_conductivity(mesh, TEMPS)["kappa"])
    ph.wigner_chunk_bytes = 1  # one q per call
    err = _rel(ph.thermal_conductivity_wigner(mesh, TEMPS)["kappa_c"], base["kappa_c"])
    ph.wigner_chunk_bytes = Phonons.wigner_chunk_bytes
    one = ph.thermal_conductivity_wigner(mesh, [300.0])
    err_t = _rel(one["kappa_c"][0], base["kappa_c"][1])
    print(f"LiMnO2 2x1x1 on 2^3: one q per call vs default {err:.2e}; one temperature vs three {err_t:.2e}")
    assert err <= 1e-13 and err_t <= 1e-13
    for bad in ([-1.0], [float("nan")], None):
        with pytest.raises(ValueError, match="temperatures"):
            ph.thermal_conductivity_wigner(mesh, bad)
    no3 = Phonons(fc, sc, device="cpu", kernels=WignerSpecKernels())
    with pytest.raises(ValueError, match="third_order=True"):
        no3.thermal_conductivity_wigner(mesh, [300.0])


def test_header_chunk_limit():
    from chgnet_b200 import _lib

    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "chgnet_b200.h")).read(), flags=re.S)
    assert _lib.WIGNER_MAX_CHUNKS == int(re.search(r"#define CHG_WIGNER_MAX_CHUNKS\s+(\d+)", src).group(1))
    assert _lib.coherence_scratch_doubles(5, 7, 3) == 12 * 5 * 49 + _lib.WIGNER_MAX_CHUNKS * 3 * 6


def test_rotation_keeps_sets():
    """``rotate_sets`` mixes modes only inside a set and keeps them orthonormal."""
    g = torch.Generator().manual_seed(0)
    e = torch.linalg.qr(torch.complex(torch.randn(2, 6, 6, generator=g, dtype=torch.float64),
                                      torch.randn(2, 6, 6, generator=g, dtype=torch.float64)))[0].mT.contiguous()
    sid = torch.tensor([[0, 0, 1, 2, 2, 2], [0, 1, 2, 3, 4, 5]])
    r = rotate_sets(e, sid, torch.Generator().manual_seed(1))
    assert torch.allclose(r @ r.mH, torch.eye(6, dtype=torch.complex128).expand(2, 6, 6), atol=1e-14)
    assert torch.equal(r[1], e[1]) and torch.equal(r[0, 2], e[0, 2])
    proj = lambda x, i: x[i].mH @ x[i]  # noqa: E731  projector of a set (mode-major rows)
    assert torch.allclose(proj(r[0], [0, 1]), proj(e[0], [0, 1]), atol=1e-14)
    assert torch.allclose(proj(r[0], [3, 4, 5]), proj(e[0], [3, 4, 5]), atol=1e-14)
