"""TEST INFRASTRUCTURE — strain second-derivative fixture from the live reference (run where the reference tree exists).

Writes ``tests/golden/chgnet_0.3.0_elastic.npz``: for LiMnO2 mp-18767 and one seeded random cell, the strain-strain
block d^2E/dstrain^2 ([3,3,3,3], eV) and the position-strain block d^2E/dx dstrain ([3N,3,3], eV/A) of the
UNMODIFIED reference 0.3.0 model, E the total energy.  Both are autograd derivatives of the reference's own
``create_graph=True`` stress (reference model.py:527-535) multiplied by its own (not detached) volume / 160.21766208,
so the strain dependence of the volume cancels and the product is dE/dstrain: with respect to its strain tensor
(``BatchedGraph.strains``) and its Cartesian positions (``BatchedGraph.atom_positions``).  The reference runs in
float64 when it can and in float32 otherwise; the file records the dtype and the relative tolerance
(``<name>.rtol``, of the block's max) at which ``oracle.elastic.oracle_strain_blocks`` must reproduce both blocks.

    python oracle/make_golden_elastic.py
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
from oracle.elastic import EV_A3_TO_GPA, oracle_strain_blocks  # noqa: E402
from oracle.make_golden import GOLD, to_ref_graph  # noqa: E402
from oracle.ref_import import load_reference_model  # noqa: E402


def reference_strain_blocks(model, graph, dtype) -> tuple[np.ndarray, np.ndarray]:
    mm = sys.modules["chgnet.model.model"]
    rg = to_ref_graph(graph)
    rg.atom_frac_coord = rg.atom_frac_coord.to(dtype)
    rg.lattice = rg.lattice.to(dtype)
    rg.neighbor_image = rg.neighbor_image.to(dtype)
    bg = mm.BatchedGraph.from_graphs([rg], bond_basis_expansion=model.bond_basis_expansion,
                                     angle_basis_expansion=model.angle_basis_expansion, compute_stress=True)
    pred = model._compute(bg, compute_force=True, compute_stress=True)
    de = (pred["s"][0] * bg.volumes[0] / EV_A3_TO_GPA).reshape(-1)
    eps, x = bg.strains[0], bg.atom_positions[0]
    D = torch.stack([torch.autograd.grad(de[k], eps, retain_graph=True)[0] for k in range(9)])
    lam = torch.stack([torch.autograd.grad(de[k], x, retain_graph=True)[0].reshape(-1) for k in range(9)])
    return (D.detach().double().numpy().reshape(3, 3, 3, 3),
            lam.detach().double().numpy().T.reshape(-1, 3, 3).copy())


def main() -> None:
    warnings.filterwarnings("ignore")
    model = load_reference_model("0.3.0")
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    try:
        model = model.double()
        dtype = torch.float64
        z, frac, lat = graphgen.limno2_structure()
        reference_strain_blocks(model, graphgen.make_crystal_graph(z, frac, lat, backend="numpy"), dtype)
    except Exception as exc:  # noqa: BLE001  the reference hard-codes float32 somewhere on this path
        print("reference does not run in float64:", exc)
        model, dtype = model.float(), torch.float32
    fix: dict = {"dtype": np.array(str(dtype).replace("torch.", ""))}
    z, frac, lat = graphgen.limno2_structure()
    zr, fr, lr = graphgen.random_structure(10, 4712)
    for name, (zz, ff, ll) in (("limno2", (z, frac, lat)), ("random", (zr, fr, lr))):
        g = graphgen.make_crystal_graph(zz, ff, ll, backend="numpy")
        ref = reference_strain_blocks(model, g, dtype)
        orc = oracle_strain_blocks(sd, g)
        rel = max(np.abs(o - r).max() / np.abs(r).max() for o, r in zip(orc, ref))
        # pin at 10x the observed agreement, floored at the dtype's resolution
        rtol = max(10 * rel, 1e-10 if dtype == torch.float64 else 1e-5)
        print(f"{name}: n={len(zz)} max|D|={np.abs(ref[0]).max():.4f} max|Lambda|={np.abs(ref[1]).max():.4f}  "
              f"|oracle64 - ref|/max = {rel:.2e}  rtol {rtol:.1e}")
        fix.update({f"{name}.strain_strain": ref[0], f"{name}.internal_strain": ref[1], f"{name}.rtol": np.array(rtol),
                    f"{name}.z": np.asarray(zz), f"{name}.frac": np.asarray(ff), f"{name}.lattice": np.asarray(ll)})
    path = os.path.join(GOLD, "chgnet_0.3.0_elastic.npz")
    np.savez_compressed(path, **fix)
    print("wrote", path, "reference dtype", fix["dtype"])


if __name__ == "__main__":
    main()
