"""Time the direct LBTE solution on the device: the collision-matrix rows, the eigendecomposition and the whole
``Phonons.thermal_conductivity_lbte`` against ``Phonons.thermal_conductivity``.

    python tools/time_lbte.py [--repeats 2] [--mesh 8] [--kappa-mesh 6] [--supercell 2]

With LiMnO2 on a supercell^3 supercell (0.3.0 weights, fc3 from ``CHGNet.phonons(..., third_order=True)``): on a
mesh^3 mesh, for one target and every q1, ``chg_collision_rows`` at 300 K over the chunks the method uses (CUDA
events); ``torch.linalg.eigh`` of a symmetric fp64 matrix of the size M = N 3n of the kappa-mesh and of the mesh (CUDA
events); ``thermal_conductivity`` and ``thermal_conductivity_lbte`` at 300 K on the kappa-mesh and on the mesh (wall
clock ending in a synchronise), whose difference less eigh is the build of the collision matrix.  Prints the GPU name
and power limit first: the times belong to that card.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chgnet_b200 import graphgen  # noqa: E402
from chgnet_b200.model import CHGNet  # noqa: E402
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ  # noqa: E402
from tools.time_phonons import gpu_card, timed  # noqa: E402
from tools.time_thermal_displacements import event_ms  # noqa: E402


def eigh_ms(m: int, repeats: int) -> float:
    """torch.linalg.eigh of a random symmetric fp64 [m, m] on the device (CUDA events, ms per call)."""
    a = torch.randn(m, m, dtype=torch.float64, device="cuda")
    a = a + a.mT
    return event_ms(lambda: torch.linalg.eigh(a), repeats)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--mesh", type=int, default=8)
    ap.add_argument("--kappa-mesh", type=int, default=6)
    ap.add_argument("--supercell", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps({"gpu": gpu_card()}))
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"),
                             version="0.3.0").to("cuda")
    s = args.supercell
    ph = model.phonons(graphgen.limno2_structure(), [s, s, s], third_order=True)

    m = (args.mesh,) * 3
    temps = torch.tensor([300.0], dtype=torch.float64, device="cuda")
    mesh, nu, e, _, tets, _ = ph._three_phonon_mesh(m, None)
    n_mesh, nb = nu.shape
    target = n_mesh // 3 + 1
    chunk = ph._q1_chunk(len(temps))
    chunks = [torch.arange(a, min(a + chunk, n_mesh), dtype=torch.int32, device="cuda")
              for a in range(0, n_mesh, chunk)]
    ps = [ph._interactions(mesh, nu, e, target, q1) for q1 in chunks]
    out = torch.zeros(4, 1, nb, n_mesh, nb, dtype=torch.float64, device="cuda")
    omega = nu[target].contiguous()

    def rows():
        for q1, p in zip(chunks, ps):
            ph.kernels.collision_rows(nu, mesh, tets, target, omega, q1, p, temps, THERMAL_CUTOFF_THZ, out)

    print(json.dumps({"mesh": list(m), "bands": nb, "q1_per_call": chunk, "calls": len(chunks),
                      "chg_collision_rows_ms_per_target": event_ms(rows, args.repeats)}))
    del ps, out
    for mm in (args.kappa_mesh, args.mesh):
        size = mm**3 * nb
        print(json.dumps({"eigh_M": size, "eigh_ms": eigh_ms(size, args.repeats)}))
    for mm in (args.kappa_mesh, args.mesh):
        km = (mm,) * 3
        rta, t_rta = timed(lambda: ph.thermal_conductivity(km, [300.0]), 1)
        res, t_lbte = timed(lambda: ph.thermal_conductivity_lbte(km, [300.0]), 1)
        print(json.dumps({"kappa_mesh": list(km), "thermal_conductivity_s": t_rta, "thermal_conductivity_lbte_s": t_lbte,
                          "kappa_lbte_300K_diag_W_per_mK": np.diag(res["kappa"][0]).tolist(),
                          "kappa_rta_300K_diag_W_per_mK": np.diag(res["kappa_rta"][0]).tolist(),
                          "n_dropped": res["n_dropped"].tolist(), "min_eigenvalue": res["min_eigenvalue"].tolist(),
                          "n_imaginary": res["n_imaginary"]}))


if __name__ == "__main__":
    main()
