"""Time CHGNet.predict_hessian against central finite differences of the forces on the same model.

    python tools/time_hessian.py [--batch-size 16] [--repeats 3]

For LiMnO2 2x2x2 (64 atoms) and 3x3x3 (216 atoms, 0.3.0 weights): the analytic Hessian (synchronised wall clock
after a warm-up call) and finite differences over 6N force calls through StaticGraphEvaluator at a 0.01 A step
(phonopy's default), and max|H_analytic - H_FD|.  Prints the GPU name and power limit first: the times belong to
that card.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chgnet_b200 import graphgen  # noqa: E402
from chgnet_b200.model import CHGNet  # noqa: E402


def gpu_card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def fd_hessian(model, z, frac, lat, step: float) -> np.ndarray:
    """-(F(x + h e_c) - F(x - h e_c)) / 2h per column c, positions moved in Cartesian space, graph fixed."""
    g = graphgen.make_crystal_graph(z, frac, lat)
    ev = model.static_evaluator(g, task="ef")
    n = len(z)
    cart = frac @ lat
    inv = np.linalg.inv(lat)
    h = np.empty((3 * n, 3 * n))
    for c in range(3 * n):
        f = []
        for sgn in (1.0, -1.0):
            x = cart.copy()
            x[c // 3, c % 3] += sgn * step
            ev.update(frac=x @ inv)
            f.append(ev()["f"].astype(np.float64).reshape(-1))
        h[:, c] = -(f[0] - f[1]) / (2 * step)
    return h


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
    ap.add_argument("--step", type=float, default=0.01)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_hessian.py needs a CUDA device")
    print(json.dumps({"card": gpu_card()}))
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    for sc in (2, 3):
        z, frac, lat = graphgen.limno2_structure((sc, sc, sc))
        g = graphgen.make_crystal_graph(z, frac, lat)
        h_an, t_an, t_an_med = timed(lambda: model.predict_hessian(g, batch_size=a.batch_size), a.repeats)
        h_fd, t_fd, t_fd_med = timed(lambda: fd_hessian(model, z, frac, lat, a.step), 1)
        scale = float(np.abs(h_an).max())
        print(json.dumps({
            "cell": f"LiMnO2 {sc}x{sc}x{sc}", "n_atoms": len(z), "batch_size": a.batch_size,
            "analytic_s_min": round(t_an, 4), "analytic_s_median": round(t_an_med, 4),
            "fd_s": round(t_fd, 4), "fd_force_calls": 6 * len(z), "fd_step_A": a.step,
            "speedup": round(t_fd / t_an, 2), "max_abs_H": round(scale, 4),
            "max_abs_H_analytic_minus_FD": float(np.abs(h_an - h_fd).max()),
            "asymmetry_analytic": float(np.abs(h_an - h_an.T).max()),
        }))


if __name__ == "__main__":
    main()
