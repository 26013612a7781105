"""Time CHGNet.predict_elastic_tensor against central finite differences of the stress on the same model.

    python tools/time_elastic.py [--batch-size 16] [--repeats 3] [--steps 1e-3 1e-4]

For LiMnO2 2x2x2 (64 atoms) and 3x3x3 (216 atoms, 0.3.0 weights): the analytic tensor with relaxed_ions=False and
with relaxed_ions=True (synchronised wall clock after a warm-up call), the clamped-ion finite-difference route (12
stress calls through StaticGraphEvaluator.update(lattice=...) at +-step Voigt strains, graph fixed) at each step,
and max|C_analytic - C_FD| per step.  Prints the GPU name and power limit first: the times belong to that card.  Needs a CUDA
device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chgnet_b200 import graphgen  # noqa: E402
from chgnet_b200.model import CHGNet  # noqa: E402

VOIGT_PAIRS = ((0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1))


def gpu_card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def fd_clamped(model, z, frac, lat, step: float) -> np.ndarray:
    """C_ab = (sigma_b(+step e_a) - sigma_b(-step e_a)) / 2 step, lattice strained at fixed fractional coordinates."""
    ev = model.static_evaluator(graphgen.make_crystal_graph(z, frac, lat), task="efs")
    c = np.empty((6, 6))
    for a, (i, j) in enumerate(VOIGT_PAIRS):
        w = np.zeros((3, 3))
        w[i, j] += 0.5
        w[j, i] += 0.5
        s = []
        for sgn in (1.0, -1.0):
            ev.update(lattice=(lat @ (np.eye(3) + sgn * step * w))[None])
            sig = ev()["s"].astype(np.float64)
            sig = 0.5 * (sig + sig.T)
            s.append(np.array([sig[p, q] for p, q in VOIGT_PAIRS]))
        c[a] = (s[0] - s[1]) / (2 * step)
    return c


def timed(fn, repeats: int):
    fn()  # warm-up: module loads, allocator, batch shapes
    torch.cuda.synchronize()
    times, out = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return out, min(times), float(np.median(times))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=float, nargs="+", default=[1e-3, 1e-4])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_elastic.py needs a CUDA device")
    warnings.simplefilter("ignore", RuntimeWarning)  # LiMnO2 has an unstable mode under 0.3.0
    print(json.dumps({"card": gpu_card()}))
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    for sc in (2, 3):
        z, frac, lat = graphgen.limno2_structure((sc, sc, sc))
        g = graphgen.make_crystal_graph(z, frac, lat)
        clamped, t_cl, t_cl_med = timed(lambda: model.predict_elastic_tensor(g, relaxed_ions=False,
                                                                           batch_size=a.batch_size), a.repeats)
        full, t_rel, t_rel_med = timed(lambda: model.predict_elastic_tensor(g, batch_size=a.batch_size), a.repeats)
        c = clamped["clamped_ion"]
        fd = {}
        for step in a.steps:
            c_fd, t_fd, _ = timed(lambda: fd_clamped(model, z, frac, lat, step), a.repeats)
            fd[f"{step:g}"] = {"s_min": round(t_fd, 4), "max_abs_C_analytic_minus_FD_GPa": round(float(np.abs(c - c_fd).max()), 3)}
        print(json.dumps({
            "cell": f"LiMnO2 {sc}x{sc}x{sc}", "n_atoms": len(z), "batch_size": a.batch_size,
            "clamped_s_min": round(t_cl, 4), "clamped_s_median": round(t_cl_med, 4),
            "relaxed_s_min": round(t_rel, 4), "relaxed_s_median": round(t_rel_med, 4),
            "fd_clamped_by_step": fd, "fd_stress_calls": 12, "max_abs_C_GPa": round(float(np.abs(c).max()), 2),
            "C_asymmetry_GPa": float(np.abs(c - c.T).max()),
            "unstable_modes": full["unstable_modes"],
            "C_relaxed_diag_GPa": [round(float(x), 2) for x in np.diag(full["relaxed_ion"])],
        }))


if __name__ == "__main__":
    main()
