"""Time isotope scattering on the device: ``chg_isotope_scattering`` per target and over a whole mesh, and
``Phonons.thermal_conductivity`` with and without ``mass_variances``.

    python tools/time_isotope.py [--repeats 20] [--mesh 8] [--supercell 2]

With LiMnO2 on a supercell^3 supercell (0.3.0 weights, fc3 from ``CHGNet.phonons(..., third_order=True)``) on a
mesh^3 mesh at 300 K: ``chg_isotope_scattering`` for one target and over the target chunks ``isotope_linewidths`` uses
for the whole mesh, inputs made beforehand (CUDA events), then ``thermal_conductivity`` without and with
``mass_variances`` alternately, twice each (wall clock ending in a synchronise).  The mass variances are illustrative
(1.5e-3 for Li, 0 for Mn, 3.4e-5 for O), not natural-abundance data.  Prints the GPU name and power limit first: the
times belong to that card.  Needs a CUDA device; there is no CPU fallback.
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
from tools.time_phonons import gpu_card  # noqa: E402
from tools.time_thermal_displacements import event_ms  # noqa: E402
from tools.time_wigner import wall_s  # noqa: E402

G = {3: 1.5e-3, 25: 0.0, 8: 3.4e-5}


class _Recording:
    """Forwards every call to the CUDA kernels and keeps the arguments of ``isotope_scattering``."""

    def __init__(self, kernels):
        self.kernels, self.calls = kernels, []

    def __getattr__(self, name):
        return getattr(self.kernels, name)

    def isotope_scattering(self, *args):
        self.calls.append(args)
        self.kernels.isotope_scattering(*args)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--mesh", type=int, default=8)
    ap.add_argument("--supercell", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps({"gpu": gpu_card()}))
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"),
                             version="0.3.0").to("cuda")
    s = args.supercell
    ph = model.phonons(graphgen.limno2_structure(), [s, s, s], third_order=True)
    g = [G[int(z)] for z in ph.cell.prim_z]
    m = (args.mesh,) * 3
    n_mesh = m[0] * m[1] * m[2]
    ph.thermal_conductivity((2, 2, 2), [300.0], mass_variances=g)  # warm-up of every kernel and eigh
    rec = _Recording(ph.kernels)
    ph.kernels = rec
    ph.isotope_linewidths(m, np.array(np.unravel_index(np.arange(n_mesh), m)).T / np.array(m), g)
    ph.kernels = rec.kernels
    calls = rec.calls
    nu, mesh, tets, e, mv, targets, omega, cut, _ = calls[0]
    one = (nu, mesh, tets, e, mv, targets[:1].clone(), omega[:1].clone(), cut, torch.empty_like(omega[:1]))

    def whole():
        for a in calls:
            rec.kernels.isotope_scattering(*a)

    nb = nu.shape[1]
    print(json.dumps({"mesh": list(m), "bands": nb, "calls": len(calls), "targets_per_call": int(targets.shape[0]),
                      "chg_isotope_scattering_ms_per_target": event_ms(lambda: rec.kernels.isotope_scattering(*one),
                                                                        args.repeats),
                      "chg_isotope_scattering_ms_per_mesh": event_ms(whole, args.repeats)}))
    times = {"thermal_conductivity_s": [], "thermal_conductivity_isotope_s": []}
    for _ in range(2):
        plain, t = wall_s(lambda: ph.thermal_conductivity(m, [300.0]))
        times["thermal_conductivity_s"].append(t)
        res, t = wall_s(lambda: ph.thermal_conductivity(m, [300.0], mass_variances=g))
        times["thermal_conductivity_isotope_s"].append(t)
    print(json.dumps({"kappa_mesh": list(m), **times,
                      "kappa_300K_diag_W_per_mK": np.diag(plain["kappa"][0]).tolist(),
                      "kappa_isotope_300K_diag_W_per_mK": np.diag(res["kappa"][0]).tolist(),
                      "max_isotope_linewidth_THz": float(np.abs(res["isotope_linewidths"]).max()),
                      "n_imaginary": res["n_imaginary"]}))


if __name__ == "__main__":
    main()
