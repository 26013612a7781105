"""fp64 numpy specification of ``chg_sample_displacements`` and ``chg_displacement_moments`` with the arguments of
``CudaKernels.sample_displacements`` and ``CudaKernels.displacement_moments``, for ``effective_force_constants(...,
kernels=EffectiveSpecKernels(), device="cpu")``.  ``normal_variates`` is the counter-based generator on its own."""
from __future__ import annotations

import numpy as np
import torch

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(x: np.ndarray) -> np.ndarray:
    """splitmix64 of uint64 ``x`` (elementwise, wrapping)."""
    with np.errstate(over="ignore"):
        z = x.astype(np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def normal_variates(seed: int, iteration: int, samples, n_modes: int) -> np.ndarray:
    """[len(samples), n_modes] standard normals xi(seed, iteration, s, lam): Box-Muller on r = h(h(h(h(seed) +
    iteration) + s) + lam), u1 = ((r >> 11) + 1) 2^-53, u2 = (h(r) >> 11) 2^-53, xi = sqrt(-2 ln u1) cos(2 pi u2)."""
    with np.errstate(over="ignore"):
        h = splitmix64(np.array([seed], dtype=np.uint64)) + np.uint64(iteration)
        h = splitmix64(splitmix64(h)[0] + np.asarray(samples, dtype=np.uint64))  # [S]
        r = splitmix64(h[:, None] + np.arange(n_modes, dtype=np.uint64)[None, :])
    u1 = ((r >> np.uint64(11)) + np.uint64(1)).astype(np.float64) * 2.0**-53
    u2 = (splitmix64(r) >> np.uint64(11)).astype(np.float64) * 2.0**-53
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def sample_draws(evecs, amp, inv_sqrt_m, seed, iteration, first_sample, n_samples) -> np.ndarray:
    """[M, N, 3] the unrounded fp64 draws d[s] = M^-1/2 sum_lam e_lam amp_lam xi(seed, iteration, s, lam)."""
    e = np.asarray(evecs, dtype=np.float64)
    xi = normal_variates(seed, iteration, np.arange(first_sample, first_sample + n_samples), e.shape[0])
    d = (xi * np.asarray(amp)[None, :]) @ e
    return (d * np.repeat(np.asarray(inv_sqrt_m), 3)[None, :]).reshape(n_samples, -1, 3)


class EffectiveSpecKernels:
    """Drop-in for the two ``CudaKernels`` methods of ``effective_force_constants``, on host tensors."""

    name = "spec"

    def sample_displacements(self, evecs, amp, inv_sqrt_m, frac_ref, lattice, inv_lattice, seed, iteration,
                             first_sample, frac, u):
        m = u.shape[0]
        d = sample_draws(evecs.cpu().numpy(), amp.cpu().numpy(), inv_sqrt_m.cpu().numpy(), seed, iteration,
                         first_sample, m)
        ref = frac_ref.cpu().numpy()
        f32 = (ref[None] + d @ inv_lattice.cpu().numpy()).astype(np.float32)
        du = f32.astype(np.float64) - ref.astype(np.float32).astype(np.float64)[None]
        frac.copy_(torch.from_numpy(f32.reshape(-1, 3)))
        u.copy_(torch.from_numpy(du @ lattice.cpu().numpy()))

    def displacement_moments(self, u, force, f0, perm, acc):
        """Plain loops over the samples, translations and atoms; each sample's sums are added to acc in turn."""
        uu, ff, f0n, p = u.cpu().numpy(), force.cpu().numpy(), f0.cpu().numpy(), perm.cpu().numpy()
        m, n = uu.shape[:2]
        n_cells = p.shape[0]
        n_prim = n // n_cells
        n_g = 9 * n_prim * n
        out = acc.cpu().numpy().copy()
        for s in range(m):
            df = ff[s] - f0n
            g = np.zeros((n_prim, 3, n, 3))
            b = np.zeros((n_prim, 3, n, 3))
            for k in range(n_prim):
                a = p[:, k * n_cells]  # [n_cells] T_l(p2s k)
                g[k] = np.einsum("lx,ljy->xjy", uu[s][a], uu[s][p])
                b[k] = np.einsum("lx,ljy->xjy", df[a], uu[s][p])
            out[:n_g] += g.reshape(-1)
            out[n_g : 2 * n_g] += b.reshape(-1)
            out[2 * n_g] += float((df * df).sum())
            out[2 * n_g + 1] += float((f0n * uu[s]).sum())
        acc.copy_(torch.from_numpy(out))
