"""TEST INFRASTRUCTURE — Hessian fixture from the live reference (run where the reference tree exists).

Writes ``tests/golden/chgnet_0.3.0_hessian.npz``: d^2E/dx dx ([3N,3N], eV/A^2, total energy, fixed cell) of
the UNMODIFIED reference 0.3.0 model on LiMnO2 mp-18767 and on one seeded random cell, taken by autograd of
the reference's own ``create_graph=True`` forces (reference model.py:517-524) with respect to its
``BatchedGraph.atom_positions``.  The reference runs in float64 when it can (``model.double()`` + float64
graphs) and in float32 otherwise; the file records the dtype and the relative tolerance
(``<name>.rtol``, of max|H|) at which the fp64 oracle must reproduce each Hessian.

    python oracle/make_golden_hessian.py
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chgnet_b200 import graphgen  # noqa: E402
from oracle.hessian import oracle_hessian  # noqa: E402
from oracle.make_golden import GOLD, to_ref_graph  # noqa: E402
from oracle.ref_import import load_reference_model  # noqa: E402


def reference_hessian(model, graph, dtype) -> np.ndarray:
    mm = sys.modules["chgnet.model.model"]
    rg = to_ref_graph(graph)
    rg.atom_frac_coord = rg.atom_frac_coord.to(dtype).requires_grad_(True)  # as the reference's converter does
    rg.lattice = rg.lattice.to(dtype)
    rg.neighbor_image = rg.neighbor_image.to(dtype)
    bg = mm.BatchedGraph.from_graphs([rg], bond_basis_expansion=model.bond_basis_expansion,
                                     angle_basis_expansion=model.angle_basis_expansion, compute_stress=False)
    pred = model._compute(bg, compute_force=True, compute_stress=False)
    f = pred["f"][0].reshape(-1)
    x = bg.atom_positions[0]
    return torch.stack([torch.autograd.grad(-f[k], x, retain_graph=True)[0].reshape(-1)
                        for k in range(f.numel())]).detach().double().numpy()


def main() -> None:
    warnings.filterwarnings("ignore")
    model = load_reference_model("0.3.0")
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    try:
        model = model.double()
        dtype = torch.float64
        z, frac, lat = graphgen.limno2_structure()
        reference_hessian(model, graphgen.make_crystal_graph(z, frac, lat, backend="numpy"), dtype)
    except Exception as exc:  # noqa: BLE001  the reference hard-codes float32 somewhere on this path
        print("reference does not run in float64:", exc)
        model, dtype = model.float(), torch.float32
    fix: dict = {"dtype": np.array(str(dtype).replace("torch.", ""))}
    z, frac, lat = graphgen.limno2_structure()
    zr, fr, lr = graphgen.random_structure(10, 4711)
    for name, (zz, ff, ll) in (("limno2", (z, frac, lat)), ("random", (zr, fr, lr))):
        g = graphgen.make_crystal_graph(zz, ff, ll, backend="numpy")
        h_ref = reference_hessian(model, g, dtype)
        h_orc = oracle_hessian(sd, g)
        scale = np.abs(h_ref).max()
        rel = np.abs(h_orc - h_ref).max() / scale
        # pin at 10x the observed agreement, floored at the dtype's resolution
        rtol = max(10 * rel, 1e-10 if dtype == torch.float64 else 1e-5)
        print(f"{name}: n={len(zz)} max|H|={scale:.4f}  |oracle64 - ref|/max|H| = {rel:.2e}  rtol {rtol:.1e}")
        fix.update({f"{name}.hessian": h_ref, f"{name}.rtol": np.array(rtol), f"{name}.z": np.asarray(zz),
                    f"{name}.frac": np.asarray(ff), f"{name}.lattice": np.asarray(ll)})
    path = os.path.join(GOLD, "chgnet_0.3.0_hessian.npz")
    np.savez_compressed(path, **fix)
    print("wrote", path, "reference dtype", fix["dtype"])


if __name__ == "__main__":
    main()
