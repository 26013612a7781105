"""fp64 torch specification of ``chg_coherence_conductivity`` with the arguments of ``CudaKernels.coherence_conductivity``.

``WignerSpecKernels`` adds it to ``ThreePhononSpecKernels`` (tests/three_phonon_kernels.py), so that
``Phonons(..., fc3=..., device="cpu", kernels=WignerSpecKernels())`` runs ``thermal_conductivity_wigner`` on the host.
``velocity_operator``, ``coherence_pairs`` and ``coherence_sum`` are module functions so that the tests can use them on
their own.  ``same_set_pairs=True`` plants the bug the tests must catch: it also sums the pairs s != s' inside a
degenerate set, whose terms depend on the basis eigh picks in the set.  ``rotation_seed`` rotates the eigenvectors of
every degenerate set by a random unitary before V is formed (the basis-invariance tests).
"""
from __future__ import annotations

import math

import torch

from chgnet_b200.phonons import THZ_PER_SQRT_EV_A2_AMU
from three_phonon_kernels import ThreePhononSpecKernels

# Voigt order of the 6 independent components, and their places in [3, 3]
VOIGT = ((0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1))


def velocity_operator(freqs, eigvecs, ddyn):
    """V [Q, 3, nb, nb] complex128 (THz A): V_a[s, s'] = c^2 <e_s| ddyn[a] |e_s'> / (|nu_s| + |nu_s'|) (0 where both
    are 0), c = ``THZ_PER_SQRT_EV_A2_AMU``, for freqs [Q, nb], mode-major eigvecs [Q, mode, nb] and ddyn
    [Q, 3, nb, nb]."""
    e = eigvecs.to(torch.complex128)
    m = e.conj()[:, None] @ ddyn.to(torch.complex128) @ e.mT[:, None]
    a = freqs.to(torch.float64).abs()
    den = (a[:, :, None] + a[:, None, :])[:, None]
    return torch.where(den > 0, THZ_PER_SQRT_EV_A2_AMU**2 * m / torch.where(den > 0, den, 1.0), 0.0)


def coherence_pairs(freqs, set_id, gamma, cutoff_thz, same_set_pairs=False):
    """[T, Q, nb, nb] bool: the ordered pairs (s, s') whose two modes have nu >= ``cutoff_thz`` and Gamma > 0 and lie
    in different degenerate sets (``same_set_pairs``: any s != s')."""
    keep = (freqs >= cutoff_thz)[None] & (gamma > 0)  # [T, Q, nb]
    pair = keep[..., :, None] & keep[..., None, :]
    if same_set_pairs:
        eye = torch.eye(freqs.shape[1], dtype=torch.bool, device=freqs.device)
        return pair & ~eye
    return pair & (set_id[:, :, None] != set_id[:, None, :])[None]


def coherence_sum(freqs, vel, heat_capacity, gamma, pairs):
    """[T, 3, 3]: the unscaled pair sum of DESIGN.md section 12.10 over the ``pairs`` [T, Q, nb, nb],
    (nu_s + nu_s') / 4 (C_s / nu_s + C_s' / nu_s') Re(V_a[s, s'] V_b[s', s]) (G_s + G_s') / (2 pi [(nu_s - nu_s')^2
    + (G_s + G_s')^2]) with V_b[s', s] = conj(V_b[s, s'])."""
    f64 = torch.float64
    nu = freqs.to(f64)
    safe = torch.where(nu > 0, nu, 1.0)
    cn = heat_capacity.to(f64) / safe[None]  # [T, Q, nb]
    g = gamma.to(f64)
    gs = g[..., :, None] + g[..., None, :]
    dn = nu[:, :, None] - nu[:, None, :]
    w = 0.25 * (nu[:, :, None] + nu[:, None, :])[None] * (cn[..., :, None] + cn[..., None, :]) * gs
    w = w / (2 * math.pi * (dn[None] ** 2 + gs**2))
    w = torch.where(pairs, w, 0.0)
    out = torch.zeros(w.shape[0], 3, 3, dtype=f64, device=freqs.device)
    for a, b in VOIGT:
        prod = (vel[:, a] * vel[:, b].conj()).real  # [Q, nb, nb]
        out[:, a, b] = out[:, b, a] = torch.einsum("tqij,qij->t", w, prod)
    return out


def rotate_sets(eigvecs, set_id, generator):
    """Mode-major eigvecs [Q, mode, nb] with the modes of every degenerate set (``set_id`` [Q, nb]) replaced by a random
    unitary combination of themselves (Haar, from ``generator``)."""
    out = eigvecs.clone()
    for q in range(eigvecs.shape[0]):
        for sid in torch.unique(set_id[q]):
            idx = torch.nonzero(set_id[q] == sid)[:, 0]
            if len(idx) < 2:
                continue
            k = len(idx)
            z = torch.complex(torch.randn(k, k, generator=generator, dtype=torch.float64),
                              torch.randn(k, k, generator=generator, dtype=torch.float64))
            u = torch.linalg.qr(z)[0].to(eigvecs.device)
            out[q, idx] = u.mT @ eigvecs[q, idx]
    return out


class WignerSpecKernels(ThreePhononSpecKernels):
    """``ThreePhononSpecKernels`` with the specification of ``chg_coherence_conductivity``."""

    def __init__(self, *, same_set_pairs: bool = False, rotation_seed: int | None = None, axes_reversed: bool = False):
        super().__init__(axes_reversed=axes_reversed)
        self.same_set_pairs = same_set_pairs
        self.rotation = None if rotation_seed is None else torch.Generator().manual_seed(rotation_seed)

    def coherence_conductivity(self, freqs, eigvecs, ddyn, set_id, heat_capacity, gamma, cutoff_thz, kappa):
        """kappa += ``coherence_sum`` over ``coherence_pairs`` with the ``velocity_operator`` of the call."""
        e = eigvecs if self.rotation is None else rotate_sets(eigvecs, set_id, self.rotation)
        vel = velocity_operator(freqs, e, ddyn)
        pairs = coherence_pairs(freqs, set_id, gamma, cutoff_thz, self.same_set_pairs)
        kappa += coherence_sum(freqs, vel, heat_capacity, gamma, pairs)
