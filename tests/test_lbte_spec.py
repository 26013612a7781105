"""CPU (fp64): the collision matrix and the LBTE thermal conductivity of chgnet_b200.phonons with the specification of
``chg_collision_rows`` (tests/lbte_kernels.py).

* the matrix against a plain loop over (q, q1, class) written from the process table of DESIGN.md section 12.8, which
  the time-reversal bug fails;
* on the spring crystal with cubic chain terms: couplings only between modes polarised along the same axis, and the
  two-column form equal to phonopy's "vertex column doubled" form;
* the RTA limit (S = 0), kappa_rta bitwise ``thermal_conductivity``'s kappa, the classical limit;
* detailed balance and the energy mode before symmetrisation, gated at their measured values, and the class-1 sign bug;
* the pseudo-inverse against a direct solve, chunking, temperature groups, symmetry, T = 0 and input errors."""
import math

import numpy as np
import pytest
import torch

from chgnet_b200.phonons import (H_OVER_KB_K_PER_THZ, KAPPA_W_PER_MK, THERMAL_CUTOFF_THZ, Phonons,
                                 _degenerate_operators)
from lbte_kernels import TWO_PI_K, LbteSpecKernels, inverse_sinh
from phonon_cells import limno2_211, springs
from test_three_phonon_spec import KS, _chain_fc3, _random_symmetric_fc3
from three_phonon_kernels import ThreePhononSpecKernels, vertex_weights

CUT = THERMAL_CUTOFF_THZ
f64 = torch.float64


class _ZeroRows(LbteSpecKernels):
    def collision_rows(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, out):
        out[:, :, :, q1.long()] = 0.0


class _HalfRows(LbteSpecKernels):
    def collision_rows(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, out):
        super().collision_rows(freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, out)
        out[:, :, :, q1.long()] *= 0.5


def _springs(mesh_kernels=LbteSpecKernels()):
    ph, _ = springs((3, 3, 3), ks=KS)
    return Phonons(ph.force_constants, ph.cell, fc3=_chain_fc3(ph.cell), device="cpu", kernels=mesh_kernels)


def _limno2(weights030, kernels=None):
    sc, _, fc = limno2_211(weights030)
    _, compact = _random_symmetric_fc3(sc, 3)
    return Phonons(fc, sc, fc3=compact, device="cpu", kernels=kernels or LbteSpecKernels())


def _loop_matrix(ph, mesh, temps):
    """S [T, N 3n, N 3n] by a loop over (q, q1, class) with explicit mesh-index arithmetic: each term of P feeds its
    two other modes c with u_q u_c 2 pi K P g / s(nu_o), o the third mode."""
    mesh_t, nu, _, _, tets, _ = ph._three_phonon_mesh(mesh, None)
    n_mesh, nb = nu.shape
    t = torch.as_tensor(np.array(temps))
    inv_s = inverse_sinh(nu, t, CUT).numpy()  # [N, 3n, T]
    nu_np = nu.numpy()
    size = np.array(mesh_t)
    coord = lambda i: np.array(np.unravel_index(i, mesh_t))  # noqa: E731
    index = lambda c: int(np.ravel_multi_index(tuple(np.asarray(c) % size), mesh_t))  # noqa: E731
    s = np.zeros((len(temps), n_mesh, nb, n_mesh, nb))
    q1_all = torch.arange(n_mesh, dtype=torch.int32)
    for q in range(n_mesh):
        p = ph._interaction_strength(mesh, coord(q) / size)  # [N, l, l1, l2]
        w = vertex_weights(nu, mesh_t, tets, q, nu[q], q1_all, CUT).numpy()  # [N, l, l1, l2, 3]
        for q1 in range(n_mesh):
            q2 = index(coord(q) - coord(q1))
            mq1, mq2 = index(-coord(q1)), index(-coord(q2))
            assert np.allclose(nu_np[mq1], nu_np[q1], atol=1e-9)
            # (class, weight, [(column q, column bands side, u_q u_c, mode o (q, side))])
            table = [
                (0, [(q1, 1, -1.0, (q2, 2)), (q2, 2, -1.0, (q1, 1))]),   # (a) q -> q1 + q2
                (1, [(mq1, 1, +1.0, (q2, 2)), (q2, 2, -1.0, (mq1, 1))]),  # (b) q + (-q1) -> q2
                (2, [(q1, 1, -1.0, (mq2, 2)), (mq2, 2, +1.0, (q1, 1))]),  # (c) q + (-q2) -> q1
            ]
            for cls, feeds in table:
                term = TWO_PI_K * p[q1] * w[q1, ..., cls]  # [l, l1, l2]
                for col_q, side, u, (oq, oside) in feeds:
                    o = inv_s[oq]  # [3n, T], indexed by the band of o
                    if side == 1:  # column (col_q, l1), o carries l2
                        s[:, q, :, col_q, :] += u * np.einsum("lab,bt->tla", term, o)
                    else:  # column (col_q, l2), o carries l1
                        s[:, q, :, col_q, :] += u * np.einsum("lab,at->tlb", term, o)
    return s.reshape(len(temps), n_mesh * nb, n_mesh * nb)


@pytest.mark.parametrize("cell,mesh", [("springs", (3, 3, 3)), ("limno2", (3, 1, 1))])
def test_matrix_against_loop(cell, mesh, weights030):
    temps = [300.0, 1000.0]
    make = (lambda k: _springs(k)) if cell == "springs" else (lambda k: _limno2(weights030, k))
    ph = make(LbteSpecKernels())
    want = _loop_matrix(ph, mesh, temps)
    got = ph._collision_matrix(mesh, temps)[0].numpy()
    scale = np.abs(want).max()
    err = np.abs(got - want).max() / scale
    bug = make(LbteSpecKernels(time_reversal=False))._collision_matrix(mesh, temps)[0].numpy()
    err_bug = np.abs(bug - want).max() / scale
    print(f"{cell} on {mesh}: collision rows + gather vs plain loop {err:.2e} of max|S| {scale:.3e}; "
          f"without time reversal {err_bug:.2e}")
    assert scale > 0 and err <= 1e-12
    assert err_bug >= 1e-3


def test_spring_crystal_axes_and_doubled_form():
    ph = _springs()
    mesh, temps = (3, 3, 3), [300.0]
    s = ph._collision_matrix(mesh, temps)[0][0].numpy()
    mesh_t, nu, e, _, tets, _ = ph._three_phonon_mesh(mesh, None)
    n_mesh, nb = nu.shape
    axis = e.abs().argmax(-1).reshape(-1).numpy()  # mode-major: the axis of each mode
    cross = axis[:, None] != axis[None, :]
    assert np.all(s[cross] == 0.0) and np.abs(s[~cross]).max() > 0
    # phonopy's form: the vertex column only, doubled
    t = torch.tensor(temps, dtype=f64)
    size = np.array(mesh_t)
    coords = np.stack(np.unravel_index(np.arange(n_mesh), mesh_t), 1)
    flat = lambda c: torch.as_tensor(np.ravel_multi_index(tuple((c % size).T), mesh_t))  # noqa: E731
    q1 = torch.arange(n_mesh, dtype=torch.int32)
    worst, scale = 0.0, 0.0
    for target in range(n_mesh):
        r = torch.zeros(4, 1, nb, n_mesh, nb, dtype=f64)
        p = ph._interactions(mesh_t, nu, e, target, q1)
        ph.kernels.collision_rows(nu, mesh_t, tets, target, nu[target].contiguous(), q1, p, t, CUT, r)
        two = r[0] + r[1][:, :, flat(-coords)] + r[2][:, :, flat(coords[target] - coords)]
        two = two + r[3][:, :, flat(coords[target] + coords)]
        doubled = 2 * (r[0] + r[1][:, :, flat(-coords)])
        worst = max(worst, float((two - doubled).abs().max()))
        scale = max(scale, float(two.abs().max()))
    print(f"spring crystal 3^3: two-column form vs vertex column doubled {worst / scale:.2e} of max {scale:.3e}")
    assert scale > 0 and worst <= 1e-12 * scale


def test_rta_limit(weights030):
    mesh, temps = (2, 2, 2), [0.0, 300.0, 1000.0]
    ph = _limno2(weights030, _ZeroRows())
    r = ph.thermal_conductivity_lbte(mesh, temps)
    err = np.abs(r["kappa"] - r["kappa_rta"]).max() / np.abs(r["kappa_rta"]).max()
    print(f"LiMnO2 2x1x1 on 2^3, S = 0: kappa vs kappa_rta {err:.2e}")
    assert err <= 1e-13
    rta = ph.thermal_conductivity(mesh, temps)
    assert np.array_equal(r["kappa_rta"], rta["kappa"])
    for k in ("frequencies", "linewidths", "group_velocities", "heat_capacity", "n_zero_linewidth"):
        assert np.array_equal(r[k], rta[k])


def _omega_raw(ph, mesh, temps):
    """diag(4 pi Gamma) + (S + S^T) / 2 on the kept modes of each temperature, without degenerate averaging."""
    s, gamma, kept = ph._collision_matrix(mesh, temps)
    out = []
    for i in range(len(temps)):
        k = kept[i]
        om = torch.diag(4 * math.pi * gamma[i].reshape(-1)[k]) + 0.5 * (s[i] + s[i].mT)[k][:, k]
        out.append(om)
    return out


def test_classical_limit(weights030):
    ph = _limno2(weights030)
    mesh, big = (2, 2, 2), [1e5, 2e5]
    om = _omega_raw(ph, mesh, big)
    assert om[0].shape == om[1].shape
    nu_max = float(ph._three_phonon_mesh(mesh, None)[1].max())
    tol = (H_OVER_KB_K_PER_THZ * nu_max / big[0]) ** 2
    err = float((om[0] / big[0] - om[1] / big[1]).abs().max() / (om[1] / big[1]).abs().max())
    r = ph.thermal_conductivity_lbte(mesh, big)
    tk = r["kappa"] * np.array(big)[:, None, None]
    err_k = np.abs(tk[0] - tk[1]).max() / np.abs(tk[1]).max()
    print(f"LiMnO2 2x1x1 on 2^3 at 1e5 and 2e5 K: Omega / T {err:.2e}, T kappa {err_k:.2e}, bound (h nu_max / k T)^2 "
          f"{tol:.2e}")
    assert err <= tol and err_k <= tol


def _balance(ph, mesh, temp=300.0):
    """(||S - S^T||_F / ||S||_F, ||Omega psi|| / (||Omega||_2 ||psi||)) before symmetrisation, psi = nu / s(nu)."""
    s, gamma, kept = ph._collision_matrix(mesh, [temp])
    k = kept[0]
    sk = s[0][k][:, k]
    nu = ph._three_phonon_mesh(mesh, None)[1].reshape(-1)[k]
    om = torch.diag(4 * math.pi * gamma[0].reshape(-1)[k]) + sk
    psi = nu * inverse_sinh(nu, torch.tensor([temp], dtype=f64), CUT)[:, 0]
    return (float((sk - sk.mT).norm() / sk.norm()),
            float((om @ psi).norm() / (torch.linalg.matrix_norm(om, 2) * psi.norm())))


# measured (the asymmetry of S, the energy-mode residual) and a 5 % margin; DESIGN.md section 12.8 explains why the
# tetrahedron weights leave S entrywise far from symmetric on these meshes
BALANCE = {"springs": ((5, 5, 5), 0.6030, 0.01102), "limno2": ((2, 2, 2), 1.0368, 0.04901)}


@pytest.mark.parametrize("cell", ["springs", "limno2"])
def test_detailed_balance_and_energy_mode(cell, weights030):
    mesh, asym, resid = BALANCE[cell]
    make = (lambda k: _springs(k)) if cell == "springs" else (lambda k: _limno2(weights030, k))
    a, e = _balance(make(LbteSpecKernels()), mesh)
    a_bug, e_bug = _balance(make(LbteSpecKernels(class1_sign=-1.0)), mesh)
    print(f"{cell} on {mesh} at 300 K: ||S - S^T|| / ||S|| {a:.4e}, energy-mode residual {e:.4e}; class-1 sign "
          f"flipped {a_bug:.4e}, {e_bug:.4e}")
    assert a <= 1.05 * asym and e <= 1.05 * resid
    assert e_bug >= 5 * 1.05 * resid


def test_solver_chunking_groups_and_errors(weights030):
    mesh, temps = (2, 2, 2), [0.0, 300.0, 1000.0]
    ph = _limno2(weights030, _HalfRows())
    r = ph.thermal_conductivity_lbte(mesh, temps)
    k = r["kappa"]
    assert np.all(k[0] == 0) and np.all(r["n_dropped"] == 0)
    assert np.abs(k - k.transpose(0, 2, 1)).max() <= 1e-13 * np.abs(k).max()
    # the same kappa by a direct solve of the averaged, symmetrised matrix
    s, gamma, kept = ph._collision_matrix(mesh, temps)
    mesh_t, nu, _, _, _, _ = ph._three_phonon_mesh(mesh, None)
    avg = torch.block_diag(*_degenerate_operators(nu))
    vol = abs(float(np.linalg.det(ph.cell.prim_lattice)))
    x = (torch.as_tensor(r["heat_capacity"]).sqrt()[..., None] * torch.as_tensor(r["group_velocities"])[None])
    worst = 0.0
    for i in (1, 2):
        sa = (avg @ s[i]) @ avg
        om = torch.diag(4 * math.pi * gamma[i].reshape(-1)) + 0.5 * (sa + sa.mT)
        kk = kept[i]
        xi = x[i].reshape(-1, 3)[kk]
        want = xi.mT @ torch.linalg.solve(om[kk][:, kk], xi) * (KAPPA_W_PER_MK / (nu.shape[0] * vol))
        worst = max(worst, float((torch.as_tensor(k[i]) - want).abs().max() / want.abs().max()))
    print(f"LiMnO2 2x1x1 on 2^3, S / 2: pseudo-inverse vs solve {worst:.2e}; kappa(300 K) diag {np.diag(k[1])}")
    assert worst <= 1e-12
    ph = _limno2(weights030)
    base = ph.thermal_conductivity_lbte(mesh, temps)
    ph.ph3_chunk_bytes = 1  # one q1 per call
    err = np.abs(ph.thermal_conductivity_lbte(mesh, temps)["kappa"] - base["kappa"]).max() / np.abs(base["kappa"]).max()
    ph.ph3_chunk_bytes = Phonons.ph3_chunk_bytes
    m0 = int((base["frequencies"] >= CUT).sum())
    ph.lbte_matrix_bytes = 8 * m0 * m0  # one temperature per group
    grouped = ph.thermal_conductivity_lbte(mesh, temps)
    print(f"LiMnO2 2x1x1 on 2^3: one q1 per call vs default {err:.2e}; min eigenvalue {base['min_eigenvalue']}, "
          f"dropped {base['n_dropped']}")
    assert err <= 1e-13
    for key in ("kappa", "kappa_rta", "n_dropped", "min_eigenvalue", "linewidths"):
        assert np.array_equal(grouped[key], base[key], equal_nan=True)
    ph.lbte_matrix_bytes = 8 * m0 * m0 - 1
    with pytest.raises(ValueError, match=f"needs {8 * m0 * m0} bytes"):
        ph.thermal_conductivity_lbte(mesh, temps)
    assert np.all(ph.thermal_conductivity_lbte(mesh, [0.0])["kappa"] == 0)  # T = 0 builds no matrix
    ph.lbte_matrix_bytes = Phonons.lbte_matrix_bytes
    for bad in (float("nan"), float("inf"), -1e-8):
        with pytest.raises(ValueError, match="pinv_cutoff"):
            ph.thermal_conductivity_lbte(mesh, temps, pinv_cutoff=bad)
    for bad in ([-1.0], [float("nan")]):
        with pytest.raises(ValueError, match="temperatures"):
            ph.thermal_conductivity_lbte(mesh, bad)
    no3 = Phonons(ph.force_constants, ph.cell, device="cpu", kernels=ThreePhononSpecKernels())
    with pytest.raises(ValueError, match="third_order=True"):
        no3.thermal_conductivity_lbte(mesh, [300.0])
