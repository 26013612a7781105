"""TEST INFRASTRUCTURE — strain second derivatives: kernel specification and the fp64 oracle elastic tensors.

* ``ElasticSpecKernels``: ``HessianSpecKernels`` plus the torch specification of ``chg_edge_tangent_bwd_virial``
  (``include/chgnet_b200.h``), same argument order and accumulated outputs.  The CPU tests run
  ``Engine.second_derivatives`` on it in fp64; the ``-m gpu`` tests check the CUDA kernel against it.
* ``oracle_strain_blocks``: d^2E/dstrain^2 and the position-strain block of ``oracle/chgnet_oracle.py`` by autograd
  of its ``create_graph=True`` (``train=True``) stress and forces, task "efs", with respect to the strain tensor
  the stress was taken against (found by walking the stress graph, like the positions in ``oracle/hessian.py``).
* ``oracle_elastic``: the Voigt clamped-ion, internal-strain and relaxed-ion tensors under the conventions of
  ``CHGNet.predict_elastic_tensor``, computed independently of it (``numpy.linalg.pinv`` of the projected Hessian).

Never imported by the product path.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import chgnet_oracle as orc
from oracle.hessian import HessianSpecKernels, _grad_leaves, oracle_hessian

EV_A3_TO_GPA = orc.EV_A3_TO_GPA
# Voigt order xx, yy, zz, yz, xz, xy; direction a is the symmetric strain (E_ij + E_ji)/2 (engineering shears)
VOIGT_PAIRS = ((0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1))


def voigt_directions() -> np.ndarray:
    w = np.zeros((6, 3, 3))
    for a, (i, j) in enumerate(VOIGT_PAIRS):
        w[a, i, j] += 0.5
        w[a, j, i] += 0.5
    return w


class ElasticSpecKernels(HessianSpecKernels):
    """``HessianSpecKernels`` with the strain output of the tangent-map derivative."""

    def edge_tangent_bwd_virial(self, rvec, dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, owner,
                                force, virial):
        """``edge_tangent_bwd``'s per-edge term g_e = d/dr_e (lam_d ddist + lam_rhat . drhat), rdot fixed, scattered
        into ``force`` (force[c] -= g, force[n] += g) and summed per graph as r_e (x) g_e into ``virial`` [B,9]."""
        f64 = torch.float64
        rh, rd, mu = rhat.to(f64), drhat.to(f64), lam_rhat.to(f64)
        d, dd = dist.to(f64)[:, None], ddist.to(f64)[:, None]
        u = d2u.long()
        is_rep = u2d.long()[u] == torch.arange(len(u))
        ld = torch.where(is_rep, lam_dist.to(f64)[u], torch.zeros_like(dist, dtype=f64))[:, None]
        mr = (mu * rh).sum(dim=1, keepdim=True)
        g = ld * rd - ((mu * rd).sum(dim=1, keepdim=True) * rh + mr * rd + dd * (mu - rh * mr) / d) / d
        force.index_add_(0, center.long(), -g)
        force.index_add_(0, nbr.long(), g)
        outer = rvec.to(f64)[:, :, None] * g[:, None, :]
        virial.index_add_(0, owner.long()[center.long()], outer.reshape(-1, 9))


def _signed_volume(graph) -> torch.Tensor:
    lat = graph.lattice.detach().double()
    return torch.dot(lat[0], torch.linalg.cross(lat[1], lat[2]))  # as the oracle's stress divides by it


def oracle_strain_blocks(weights: dict, graph, args=None) -> tuple[np.ndarray, np.ndarray]:
    """(D [3,3,3,3] eV, Lambda [3N,3,3] eV/A) of one graph in fp64, strain r_e -> r_e (I + strain) at fixed fractional
    coordinates, E the total (extensive) energy:

    * D[i,j,k,l] = d^2E / dstrain_ij dstrain_kl, by autograd of dE/dstrain = stress * V / 160.21766208 (the oracle's
      stress divides by a detached V, so this is its strain gradient exactly);
    * Lambda[3m+b, i, j] = d^2E / dx_mb dstrain_ij = -dF_mb / dstrain_ij, by autograd of the forces of the same pass."""
    P = {k: torch.as_tensor(np.asarray(w)).double() for k, w in weights.items() if not k.startswith("__")}
    out = orc.forward(P, [graph], "efs", dtype=torch.float64, train=True, args=args)
    n = graph.atomic_number.shape[0]
    de = (out["s"][0] * (_signed_volume(graph) / EV_A3_TO_GPA)).reshape(-1)
    f = out["f"][0].reshape(-1)
    D, lam = np.zeros((3, 3, 3, 3)), np.zeros((3 * n, 3, 3))
    if de.grad_fn is None:
        return D, lam
    leaves = [x for x in _grad_leaves(de) if x.shape == (3, 3)]
    assert len(leaves) == 1, "expected exactly one strain tensor in the stress graph"
    eps = leaves[0]

    def rows(y):
        r = [torch.autograd.grad(y[k], eps, retain_graph=True, allow_unused=True)[0] for k in range(y.numel())]
        return np.stack([np.zeros((3, 3)) if t is None else t.detach().numpy() for t in r])

    D = rows(de).reshape(3, 3, 3, 3)
    if f.grad_fn is not None:
        lam = rows(-f)
    return D, lam


def oracle_elastic(weights: dict, graph, args=None) -> dict:
    """clamped_ion [6,6] GPa, internal_strain [3N,6] eV/A, relaxed_ion [6,6] GPa, unstable_modes, hessian [3N,3N]
    of the fp64 oracle.  C_relaxed = C - (160.21766208/V) Lambda^T H+ Lambda with H+ the pseudo-inverse (relative
    cutoff 1e-8) of the symmetrised Hessian projected off the rigid translations."""
    D, lam = oracle_strain_blocks(weights, graph, args)
    h = oracle_hessian(weights, graph, args)
    n = h.shape[0] // 3
    vol = abs(float(_signed_volume(graph)))
    w = voigt_directions()
    clamped = EV_A3_TO_GPA / vol * np.einsum("aij,ijkl,bkl->ab", w, D, w)
    lam_v = np.einsum("mij,aij->ma", lam, w)
    hs = 0.5 * (h + h.T)
    proj = np.eye(3 * n) - np.kron(np.ones((n, n)) / n, np.eye(3))
    hp = proj @ hs @ proj
    hplus = np.linalg.pinv(hp, rcond=1e-8, hermitian=True)
    evals = np.linalg.eigvalsh(hp)
    unstable = int((evals < -1e-6 * np.abs(hs).max()).sum()) if n else 0
    relaxed = clamped - EV_A3_TO_GPA / vol * lam_v.T @ hplus @ lam_v
    return dict(clamped_ion=clamped, internal_strain=lam_v, relaxed_ion=relaxed, unstable_modes=unstable, hessian=h)
