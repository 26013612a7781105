"""Time Phonons.powder_spectrum on the device, with the split between its stages.

    python tools/time_structure_factor.py [--repeats 3] [--shells 200] [--directions 1000] [--dw-mesh 20]

With the LiMnO2 2x2x2 force constants of the 0.3.0 weights (24 modes): a powder map of ``shells`` |Q| from 0.1 to
10 1/A x ``directions`` directions, 401 frequency points from -25 to 25 THz, FWHM 0.5 THz, 300 K, Debye-Waller factor
on a dw-mesh^3 mesh.  Reports the whole call (wall clock, ending in a synchronise; the Debye-Waller mesh included),
and, over the same chunk loop, D(q), ``torch.linalg.eigh``, ``chg_structure_factors`` and ``chg_broadened_spectrum``
alone (CUDA events around each stage of each chunk, summed), with the bytes each kernel must move, computed from the
shapes.  Prints the GPU name and power limit first: the times belong to that card.  Times are the fastest of
``repeats`` after a warm-up call.  Needs a CUDA device; there is no CPU fallback.
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
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ, _signed_thz, _zero_gamma_rows, fibonacci_directions  # noqa: E402
from tools.time_phonons import gpu_card, timed  # noqa: E402

# coherent scattering lengths (fm) for Li, Mn and O; any finite values time the same
B = {3: -1.90, 25: -3.73, 8: 5.80}


def stage_ms(ph, q_red, g, u, t, coef, omega, sigma, n_dir, n_shells):
    """Per-stage CUDA-event times (ms) of one pass of powder_spectrum's chunk loop, and its spectrum."""
    dev = ph.device
    n3 = 3 * len(ph.p2s)
    kcart = 2 * np.pi * (q_red + g) @ np.linalg.inv(ph.cell.prim_lattice).T
    frac = torch.as_tensor(np.ascontiguousarray(ph.cell.prim_frac)).to(dev)
    coef = torch.as_tensor(coef).to(dev)
    spec = torch.zeros(len(t), n_shells, len(omega), dtype=torch.float64, device=dev)
    chunk = max(1, min(ph.chunk_bytes // (16 * n3 * n3), ph.eigh_batch))
    marks = []
    for s in range(0, len(q_red), chunk):
        sl = slice(s, s + chunk)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        kc, gv = torch.as_tensor(kcart[sl]).to(dev), torch.as_tensor(g[sl]).to(dev)
        ev[0].record()
        d = ph.dynamical_matrices(q_red[sl])
        ev[1].record()
        lam, e = torch.linalg.eigh(d)
        nu = _signed_thz(lam)
        _zero_gamma_rows(nu, q_red[sl])
        ev[2].record()
        w = torch.empty(len(t), nu.shape[0], n3, 2, dtype=torch.float64, device=dev)
        ph.kernels.structure_factors(nu, e.mT.contiguous(), kc, gv, frac, coef, u, t, THERMAL_CUTOFF_THZ, w)
        ev[3].record()
        ph.kernels.broadened_spectrum(nu, w, s, n_dir, omega, sigma, spec)
        ev[4].record()
        marks.append(ev)
    torch.cuda.synchronize()
    names = ("dynamical_matrices", "eigh", "structure_factors", "broadened_spectrum")
    return {n: sum(ev[i].elapsed_time(ev[i + 1]) for ev in marks) for i, n in enumerate(names)}, spec, len(marks)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--shells", type=int, default=200)
    ap.add_argument("--directions", type=int, default=1000)
    ap.add_argument("--dw-mesh", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_structure_factor.py needs a CUDA device")
    print(json.dumps({"card": gpu_card()}), flush=True)
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    ph = model.phonons(graphgen.limno2_structure(), [2, 2, 2])
    n3 = 3 * len(ph.p2s)
    qm = np.linspace(0.1, 10.0, a.shells)
    omega = np.linspace(-25.0, 25.0, 401)
    temps, width, mesh = np.array([300.0]), 0.5, (a.dw_mesh,) * 3
    out, t_call = timed(lambda: ph.powder_spectrum(qm, omega, temps, B, width=width, n_directions=a.directions,
                                                   debye_waller_mesh=mesh), a.repeats)

    # the stages of the same call, on the same rows
    u = ph._debye_waller(mesh, temps)[0]
    _, t_dw = timed(lambda: ph._debye_waller(mesh, temps), a.repeats)
    kcart = (qm[:, None, None] * fibonacci_directions(a.directions)[None]).reshape(-1, 3)
    big_q = kcart @ ph.cell.prim_lattice.T / (2 * np.pi)
    g = np.floor(big_q + 0.5)
    t = torch.as_tensor(temps).cuda()
    om = torch.as_tensor(omega).cuda()
    sigma = width / (2 * np.sqrt(2 * np.log(2)))
    coef = ph._scattering_coefficients(B)
    best, spec, n_chunks = None, None, 0
    for _ in range(a.repeats + 1):
        ms, spec, n_chunks = stage_ms(ph, big_q - g, g, u, t, coef, om, sigma, a.directions, a.shells)
        best = ms if best is None else {k: min(best[k], ms[k]) for k in ms}
    n_rows, n_t = len(big_q), len(temps)
    bytes_sf = n_rows * (n3 * n3 * 16 + n3 * 8 + n_t * n3 * 16)  # eigenvectors, frequencies, (S+, S-) written
    bytes_bs = n_rows * n3 * (8 + n_t * 16)  # frequencies and (S+, S-) read
    print(json.dumps({
        "workload": {"force_constants": "LiMnO2 2x2x2, 0.3.0 weights", "modes": n3, "shells": a.shells,
                     "directions": a.directions, "rows": n_rows, "frequency_points": len(omega),
                     "temperatures": temps.tolist(), "width_thz": width, "debye_waller_mesh": list(mesh),
                     "eigh_chunks": n_chunks},
        "powder_spectrum_call_s": round(t_call, 4),
        "debye_waller_mesh_s": round(t_dw, 4),
        "stage_ms_min": {k: round(v, 3) for k, v in best.items()},
        "structure_factors_bytes": bytes_sf, "broadened_spectrum_bytes": bytes_bs,
        "structure_factors_GBps": round(bytes_sf / (best["structure_factors"] * 1e6), 1),
        "broadened_spectrum_GBps": round(bytes_bs / (best["broadened_spectrum"] * 1e6), 1),
        "n_imaginary": out["n_imaginary"], "debye_waller_n_imaginary": out["debye_waller_n_imaginary"],
        "stage_loop_equals_call": bool(np.array_equal(spec.cpu().numpy(), out["spectrum"])),
    }), flush=True)


if __name__ == "__main__":
    main()
