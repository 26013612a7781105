"""Time the frequency-resolved self-energy on the device: ``chg_self_energy_spectrum`` next to
``chg_imag_self_energy``, and the whole ``Phonons.spectral_function`` against ``Phonons.linewidths``.

    python tools/time_spectral_function.py [--repeats 3] [--mesh 8] [--points 201] [--supercell 2]

With LiMnO2 on a supercell^3 supercell (0.3.0 weights, fc3 from ``CHGNet.phonons(..., third_order=True)``): on a
mesh^3 mesh, for one target and every q1, at 0, 300 and 1 000 K, ``chg_self_energy_spectrum`` on the uniform grid of
``points`` points that ``spectral_function`` uses and ``chg_imag_self_energy`` at the target's band frequencies, over
the chunks each method uses (CUDA events, P made beforehand); the number of (item, tetrahedron, class, grid point)
weight evaluations the spectrum kernel makes; then ``spectral_function`` and ``linewidths`` at 4 q on 6^3 and on the
mesh at 300 K (wall clock ending in a synchronise).  Prints the GPU name and power limit first: the times belong to
that card.  Needs a CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from chgnet_b200 import graphgen  # noqa: E402
from chgnet_b200.model import CHGNet  # noqa: E402
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ  # noqa: E402
from tools.time_phonons import gpu_card, timed  # noqa: E402
from tools.time_thermal_displacements import event_ms  # noqa: E402


def weight_evaluations(nu, mesh, tets, target, grid) -> int:
    """The (item, tetrahedron, class, grid point) evaluations of tetra_weights in ``chg_self_energy_spectrum`` for
    the mesh index ``target``: over every mesh tetrahedron, band pair (l1, l2) and class, the grid points >= the cutoff
    in [e0, e3) of its sorted corner values, once per corner that is a live vertex (nu1 and nu2 >= the cutoff)."""
    n1, n2, n3 = mesh
    dev = nu.device
    cells = torch.arange(n1 * n2 * n3, device=dev)
    c = torch.stack([cells // (n2 * n3), (cells // n3) % n2, cells % n3], -1)  # [N, 3]
    size = torch.tensor(mesh, device=dev)
    tc = torch.tensor([target // (n2 * n3), (target // n3) % n2, target % n3], device=dev)
    corners = (c[:, None, None, :] + tets.long()[None]) % size  # [N, 6, 4, 3]
    qa = ((corners[..., 0] * n2 + corners[..., 1]) * n3 + corners[..., 2]).reshape(-1, 4)
    cb = (tc - corners) % size
    qb = ((cb[..., 0] * n2 + cb[..., 1]) * n3 + cb[..., 2]).reshape(-1, 4)
    live_grid = grid[grid >= THERMAL_CUTOFF_THZ].contiguous()
    total = 0
    for s in range(0, qa.shape[0], 512):
        a = nu[qa[s : s + 512]][:, :, :, None]  # [T, 4, l1, 1]
        b = nu[qb[s : s + 512]][:, :, None, :]  # [T, 4, 1, l2]
        live = ((a >= THERMAL_CUTOFF_THZ) & (b >= THERMAL_CUTOFF_THZ)).sum(1)  # [T, l1, l2]
        for f in (a + b, b - a, a - b):
            lo, hi = f.min(1).values.contiguous(), f.max(1).values.contiguous()
            n = torch.searchsorted(live_grid, hi) - torch.searchsorted(live_grid, lo)
            total += int((n * live).sum())
    return total


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--mesh", type=int, default=8)
    ap.add_argument("--points", type=int, default=201)
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
    temps = torch.tensor([0.0, 300.0, 1000.0], dtype=torch.float64, device="cuda")
    mesh, nu, e, _, tets, _ = ph._three_phonon_mesh(m, None)
    n_mesh, nb = nu.shape
    target = n_mesh // 3 + 1
    grid = torch.arange(args.points, dtype=torch.float64, device="cuda") * (float(2 * nu.max()) / (args.points - 1))
    omega = nu[target].contiguous()

    def chunked(chunk):
        q1s = [torch.arange(a, min(a + chunk, n_mesh), dtype=torch.int32, device="cuda")
               for a in range(0, n_mesh, chunk)]
        return q1s, [ph._interactions(mesh, nu, e, target, q1) for q1 in q1s]

    q1s, ps = chunked(ph._spectrum_q1_chunk(len(temps), args.points))
    gamma = torch.zeros(len(temps), nb, args.points, dtype=torch.float64, device="cuda")

    def spectrum():
        for q1, p in zip(q1s, ps):
            ph.kernels.self_energy_spectrum(nu, mesh, tets, target, grid, q1, p, temps, THERMAL_CUTOFF_THZ, gamma)

    t_se = event_ms(spectrum, args.repeats)
    n_se = len(q1s)
    del ps
    q1s, ps = chunked(ph._q1_chunk(len(temps)))
    g1 = torch.zeros(len(temps), nb, dtype=torch.float64, device="cuda")

    def linewidth():
        for q1, p in zip(q1s, ps):
            ph.kernels.imag_self_energy(nu, mesh, tets, target, omega, q1, p, temps, THERMAL_CUTOFF_THZ, g1)

    t_ise = event_ms(linewidth, args.repeats)
    del ps
    evals = weight_evaluations(nu, mesh, tets, target, grid)
    print(json.dumps({"mesh": list(m), "bands": nb, "points": args.points, "temperatures": temps.tolist(),
                      "chg_self_energy_spectrum_calls": n_se, "chg_self_energy_spectrum_ms_per_target": t_se,
                      "chg_imag_self_energy_calls": len(q1s), "chg_imag_self_energy_ms_per_target": t_ise,
                      "weight_evaluations": evals,
                      "weight_evaluations_per_s": evals / (t_se * 1e-3)}))
    q = [[0.0, 0.0, 0.0], [0.5, 0.5, 0.5], [0.5, 0.0, 0.0], [0.0, 0.5, 0.5]]  # on both meshes
    for mm in sorted({6, args.mesh}):
        km = (mm,) * 3
        res, t_sf = timed(lambda: ph.spectral_function(km, q, [300.0], self_energy_points=args.points), 1)
        _, t_lw = timed(lambda: ph.linewidths(km, q, [300.0]), 1)
        print(json.dumps({"mesh": list(km), "qpoints": len(q), "spectral_function_s": t_sf, "linewidths_s": t_lw,
                          "max_frequency_shift_THz": float(abs(res["frequency_shifts"]).max())}))


if __name__ == "__main__":
    main()
