"""TEST INFRASTRUCTURE — phonons: the specification of ``chg_dynamical_matrices`` and the fp64 oracle force constants.

* ``PhononSpecKernels.dynamical_matrices``: D(q) from compact force constants as explicit sums over (primitive atom,
  supercell atom) pairs and their minimum images, in fp64, chunked over q; same arguments as
  ``CudaKernels.dynamical_matrices``, so it can stand in for the CUDA kernel in ``chgnet_b200.phonons.Phonons``.
* ``oracle_compact_fcs``: the compact force constants of ``oracle/chgnet_oracle.py`` on a supercell, from
  ``oracle_hvp`` with the 3 n_prim unit directions on the ``p2s`` atoms.

Never imported by the product path.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.hessian import oracle_hvp


class PhononSpecKernels:
    """fp64 specification of the phonon kernel."""

    # pair-by-q work per chunk (complex128 elements of the [q, pair] phase sums)
    chunk_elems = 1 << 22

    def dynamical_matrices(self, fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, dyn):
        """dyn[q, 3k+a, 3k'+b] = (D + D^H)/2 with D = sum_{j: s2p[j]=k'} fc[k,j,a,b] (1/m_kj) sum_v e^{2 pi i q.v}
        inv_sqrt_m[k] inv_sqrt_m[k']."""
        f64 = torch.float64
        n_prim, n_super = fc.shape[0], fc.shape[1]
        ptr = img_ptr.long()
        mult = (ptr[1:] - ptr[:-1]).to(f64)  # [n_prim N]
        pair_of_image = torch.repeat_interleave(torch.arange(n_prim * n_super, device=fc.device), ptr[1:] - ptr[:-1])
        w = (1.0 / mult)[pair_of_image]
        m = inv_sqrt_m.to(f64)
        scale = (m[:, None] * m[None, :]).repeat_interleave(3, 0).repeat_interleave(3, 1)
        chunk = max(1, self.chunk_elems // max(1, n_prim * n_super))
        for s in range(0, qpoints.shape[0], chunk):
            q = qpoints[s : s + chunk].to(f64)
            phase = 2 * math.pi * (q @ img_vec.to(f64).T)  # [Qc, n_img]
            e = torch.complex(torch.cos(phase), torch.sin(phase)) * w
            pair = torch.zeros(q.shape[0], n_prim * n_super, dtype=torch.complex128, device=fc.device)
            pair.index_add_(1, pair_of_image, e)  # sum over the images of each pair, / multiplicity
            blocks = pair.view(-1, n_prim, n_super, 1, 1) * fc.to(torch.complex128)[None]  # [Qc, k, j, a, b]
            d = torch.zeros(q.shape[0], n_prim, n_prim, 3, 3, dtype=torch.complex128, device=fc.device)
            d.index_add_(2, s2p.long(), blocks)  # sum over the supercell atoms j of each k'
            d = d.permute(0, 1, 3, 2, 4).reshape(q.shape[0], 3 * n_prim, 3 * n_prim) * scale
            dyn[s : s + chunk] = 0.5 * (d + d.conj().transpose(1, 2))


def oracle_compact_fcs(weights: dict, graph, p2s, args=None) -> np.ndarray:
    """[n_prim, N, 3, 3] Phi[k, j, a, b] = (H e_{p2s[k], a})[j, b] of the oracle in fp64, H the Hessian of ``graph``
    (the supercell)."""
    n = graph.atomic_number.shape[0]
    n_prim = len(p2s)
    v = torch.zeros(n_prim, 3, n, 3, dtype=torch.float64)
    for a in range(3):
        v[torch.arange(n_prim), a, torch.as_tensor(np.asarray(p2s)).long(), a] = 1.0
    hv = oracle_hvp(weights, [graph] * (3 * n_prim), v.reshape(3 * n_prim * n, 3), args)
    return hv.reshape(n_prim, 3, n, 3).permute(0, 2, 1, 3).contiguous().numpy()
