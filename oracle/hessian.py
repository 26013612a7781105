"""TEST INFRASTRUCTURE — Hessian-vector products: kernel specifications and the fp64 oracle Hessian.

* ``HessianSpecKernels``: ``SpecKernels`` plus one torch function per Hessian-vector entry point of
  ``include/chgnet_b200.h`` (``chg_bond_basis_hvp``, ``chg_angle_basis_hvp``, ``chg_edge_tangent_bwd``), same
  argument order and caller-allocated (accumulated) outputs, written as explicit formulas like the rest of
  ``oracle/kernel_specs.py``.  The CPU tests run ``Engine.hessian_vector_products`` on them in fp64; the ``-m gpu``
  tests check each CUDA kernel against the function of the same name here.
* ``oracle_hessian`` / ``oracle_hvp``: d^2E/dx dx of ``oracle/chgnet_oracle.py`` by autograd of its
  ``create_graph=True`` forces (``train=True``) with respect to the Cartesian position tensors the forces were taken
  against.  ``forward`` does not return those tensors; they are the only leaves of the force graph that require a
  gradient (the weights are passed without ``requires_grad``, task "ef" has no strain), so they are found by walking
  that graph.

Never imported by the product path.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle import chgnet_oracle as orc
from oracle.kernel_specs import SpecKernels


def _rbf_d2(d, freq, rc, p):
    """d^2(basis)/dd^2 [M,R] (the second-order radial source)."""
    d = d[:, None]
    x = d / rc
    nrm = math.sqrt(2.0 / rc)
    k = freq / rc
    sn, cs = torch.sin(freq * x), torch.cos(freq * x)
    if p != 0:
        a, b, cc = -(p + 1) * (p + 2) / 2, p * (p + 2), -p * (p + 1) / 2
        env = 1 + a * x**p + b * x ** (p + 1) + cc * x ** (p + 2)
        denv = (a * p * x ** (p - 1) + b * (p + 1) * x**p + cc * (p + 2) * x ** (p + 1)) / rc
        d2env = ((a * p * (p - 1) * x ** (p - 2) if p >= 2 else 0) + b * (p + 1) * p * x ** (p - 1)
                 + cc * (p + 2) * (p + 1) * x**p) / rc**2
        inside = x < 1
        env, denv, d2env = (torch.where(inside, t, torch.zeros_like(t)) for t in (env, denv, d2env))
    else:
        env, denv, d2env = torch.ones_like(x), torch.zeros_like(x), torch.zeros_like(x)
    raw = nrm * sn / d
    draw = nrm * (k * cs / d - sn / d**2)
    d2raw = nrm * (-k * k * sn / d - 2 * k * cs / d**2 + 2 * sn / d**3)
    return d2raw * env + 2 * draw * denv + raw * d2env


class HessianSpecKernels(SpecKernels):
    """``SpecKernels`` with the Hessian-vector entry points: d/d(geometry) of T = <dE/dr, rdot>, rdot held fixed."""

    def bond_basis_hvp(self, dist, ddist, u2d, freq_ag, freq_bg, rc_ag, rc_bg, p, w3, lam_e0, lam_wag, lam_wbg, g_dist):
        """g_dist[u] += < lam W^T, d^2B/dd^2 > ddist  (second-order radial source, lam held fixed)"""
        du, ddu = dist[u2d.long()], ddist[u2d.long()]
        gb_ag = lam_e0 @ w3[0] + lam_wag @ w3[1]
        gb_bg = lam_wbg @ w3[2]
        src = (gb_ag * _rbf_d2(du, freq_ag, rc_ag, p)).sum(dim=1) + (gb_bg * _rbf_d2(du, freq_bg, rc_bg, p)).sum(dim=1)
        g_dist += src * ddu

    def angle_basis_hvp(self, rhat, drhat, ang_di, ang_dj, freq, w, lam_a0, g_rhat):
        """g_rhat += d/d(rhat_i, rhat_j) of < lam_a0, (dF/dtheta thetadot) W > with drhat held fixed
        (second-order angular source); 1 - u^2 is formed as (1 - c^2) + c^2 |rhat_i x rhat_j|^2."""
        i, j = ang_di.long(), ang_dj.long()
        ri, rj, dri, drj = rhat[i], rhat[j], drhat[i], drhat[j]
        c = 1 - 1e-6
        u = (ri * rj).sum(dim=1) * c
        q = (1 - c * c) + c * c * (torch.linalg.cross(ri, rj) ** 2).sum(dim=1)
        th_u = -1 / torch.sqrt(q)  # d theta / du
        th_uu = th_u**3 * u  # d^2 theta / du^2 = -u / (1 - u^2)^(3/2)
        ud = ((dri * rj).sum(dim=1) + (ri * drj).sum(dim=1)) * c
        thd = th_u * ud
        nf = freq.shape[0]
        gf = (lam_a0 @ w) / math.sqrt(math.pi)
        arg = torch.acos(u)[:, None] * freq[None, :]
        sn, cs = torch.sin(arg), torch.cos(arg)
        f1 = (gf[:, 1 : 1 + nf] * cs * freq).sum(dim=1) - (gf[:, 1 + nf :] * sn * freq).sum(dim=1)  # < gf, F' >
        f2 = -(gf[:, 1 : 1 + nf] * sn * freq**2).sum(dim=1) - (gf[:, 1 + nf :] * cs * freq**2).sum(dim=1)  # < gf, F'' >
        k_r = c * (f2 * thd * th_u + f1 * th_uu * ud)
        k_d = c * f1 * th_u
        g_rhat.index_add_(0, i, (k_r[:, None] * rj + k_d[:, None] * drj).to(g_rhat.dtype))
        g_rhat.index_add_(0, j, (k_r[:, None] * ri + k_d[:, None] * dri).to(g_rhat.dtype))

    def edge_tangent_bwd(self, dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, force):
        """d/dr_e of  lam_d ddist + lam_rhat . drhat  with rdot held fixed, accumulated like force_virial (force
        -= d/dx): ddist = rhat . rdot has derivative drhat; drhat = (rdot - rhat ddist)/d has the adjoint
        -[(mu . drhat) rhat + (mu . rhat) drhat + ddist (mu - rhat (rhat . mu))/d]/d."""
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


# ---------------------------------------------------------------------------------------------------------------
# fp64 oracle Hessian
# ---------------------------------------------------------------------------------------------------------------
def _grad_leaves(t: torch.Tensor) -> list[torch.Tensor]:
    """Leaf tensors (requiring a gradient) that ``t`` depends on, found by walking its autograd graph."""
    leaves, seen, stack = [], set(), [t.grad_fn]
    while stack:
        fn = stack.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        var = getattr(fn, "variable", None)  # AccumulateGrad nodes hold their leaf
        if var is not None:
            leaves.append(var)
        stack.extend(nf for nf, _ in fn.next_functions)
    return leaves


def _forces_and_positions(weights: dict, graph, args=None):
    """Oracle forces [n,3] (with their autograd graph) of one graph and the position tensor they depend on
    (None when no force depends on a position, e.g. an isolated atom)."""
    P = {k: torch.as_tensor(np.asarray(w)).double() for k, w in weights.items() if not k.startswith("__")}
    f = orc.forward(P, [graph], "ef", dtype=torch.float64, train=True, args=args)["f"][0]
    if f.grad_fn is None:
        return f, None
    n = graph.atomic_number.shape[0]
    leaves = [x for x in _grad_leaves(f) if x.shape == (n, 3)]
    assert len(leaves) <= 1, "more than one candidate position tensor in the force graph"
    return f, (leaves[0] if leaves else None)


def oracle_hessian(weights: dict, graph, args=None) -> np.ndarray:
    """[3N,3N] H[3i+a, 3j+b] = d^2E/dx_ia dx_jb of the oracle in fp64 (total energy, fixed cell)."""
    f, x = _forces_and_positions(weights, graph, args)
    f = f.reshape(-1)
    if x is None:
        return np.zeros((f.numel(), f.numel()))
    rows = [torch.autograd.grad(-f[k], x, retain_graph=True, allow_unused=True)[0] for k in range(f.numel())]
    return torch.stack([torch.zeros_like(x).reshape(-1) if r is None else r.reshape(-1) for r in rows]).detach().numpy()


def oracle_hvp(weights: dict, graphs, v: torch.Tensor, args=None) -> torch.Tensor:
    """H v per atom [N,3] (fp64) for a list of graphs (H is block-diagonal over graphs: one graph at a time)."""
    out, off = [], 0
    for g in graphs:
        n = g.atomic_number.shape[0]
        f, x = _forces_and_positions(weights, g, args)
        hv = None
        if x is not None:
            hv = torch.autograd.grad(-(f * v[off : off + n]).sum(), x, allow_unused=True)[0]
        out.append(torch.zeros(n, 3, dtype=torch.float64) if hv is None else hv.detach())
        off += n
    return torch.cat(out)
