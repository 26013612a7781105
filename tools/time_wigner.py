"""Time the Wigner coherence conductivity on the device: ``chg_coherence_conductivity`` over a whole mesh and
``Phonons.thermal_conductivity_wigner`` against ``Phonons.thermal_conductivity``.

    python tools/time_wigner.py [--repeats 20] [--mesh 8] [--supercell 2]

With LiMnO2 on a supercell^3 supercell (0.3.0 weights, fc3 from ``CHGNet.phonons(..., third_order=True)``) on a
mesh^3 mesh at 300 K: ``chg_coherence_conductivity`` over the q chunks the method uses, its inputs (dD/dQ, the
linewidths and heat capacities) already made (CUDA events), then ``thermal_conductivity`` and
``thermal_conductivity_wigner`` alternately, twice each (wall clock ending in a synchronise).  Prints the GPU name and
power limit first: the times belong to that card.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chgnet_b200 import graphgen  # noqa: E402
from chgnet_b200.model import CHGNet  # noqa: E402
from tools.time_phonons import gpu_card  # noqa: E402
from tools.time_thermal_displacements import event_ms  # noqa: E402


class _Recording:
    """Forwards every call to the CUDA kernels and keeps the arguments of ``coherence_conductivity``."""

    def __init__(self, kernels):
        self.kernels, self.calls = kernels, []

    def __getattr__(self, name):
        return getattr(self.kernels, name)

    def coherence_conductivity(self, *args):
        self.calls.append(args)
        self.kernels.coherence_conductivity(*args)


def wall_s(fn):
    """(fn(), seconds of wall clock from the call to a synchronise after it)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


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
    m = (args.mesh,) * 3
    ph.thermal_conductivity_wigner((2, 2, 2), [300.0])  # warm-up of every kernel and eigh
    rec = _Recording(ph.kernels)
    ph.kernels = rec
    res = ph.thermal_conductivity_wigner(m, [300.0])
    ph.kernels = rec.kernels
    calls = [(*a[:7], torch.zeros_like(a[7])) for a in rec.calls]

    def pair_sum():
        for a in calls:
            rec.kernels.coherence_conductivity(*a)

    nb = res["frequencies"].shape[1]
    print(json.dumps({"mesh": list(m), "bands": nb, "calls": len(calls), "q_per_call": int(calls[0][0].shape[0]),
                      "chg_coherence_conductivity_ms_per_mesh": event_ms(pair_sum, args.repeats)}))
    times = {"thermal_conductivity_s": [], "thermal_conductivity_wigner_s": []}
    for _ in range(2):
        _, t = wall_s(lambda: ph.thermal_conductivity(m, [300.0]))
        times["thermal_conductivity_s"].append(t)
        res, t = wall_s(lambda: ph.thermal_conductivity_wigner(m, [300.0]))
        times["thermal_conductivity_wigner_s"].append(t)
    print(json.dumps({"kappa_mesh": list(m), **times,
                      "kappa_p_300K_diag_W_per_mK": np.diag(res["kappa_p"][0]).tolist(),
                      "kappa_c_300K_diag_W_per_mK": np.diag(res["kappa_c"][0]).tolist(),
                      "n_imaginary": res["n_imaginary"]}))


if __name__ == "__main__":
    main()
