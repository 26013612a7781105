"""Time Phonons.joint_dos and Phonons.phase_space on the device against the fp64 specification on the host.

    python tools/time_joint_dos.py [--batch-size 16] [--repeats 3] [--jdos-mesh 20] [--meshes 8 12 16] [--host-mesh 4]

With the force constants of LiMnO2 3x3x3 (0.3.0 weights): ``joint_dos`` at 4 q-points of a jdos-mesh^3 mesh with 201
frequency points, without temperatures and with 31 from 0 to 1500 K; ``phase_space`` on each mesh^3 mesh at 0, 300
and 1000 K (wall clock, ending in a synchronise), and the ``chg_joint_dos`` kernel alone over the same target chunks
(CUDA events, on the frequencies the call uses).  Then ``phase_space`` with ``oracle/phonons.py``'s specification
on the host (``Phonons(..., device="cpu", kernels=PhononSpecKernels())``) on a host-mesh^3 mesh, with the largest
difference from the device.  Prints the GPU name and power limit first: the times belong to that card.  Times are the
fastest of ``repeats`` after a warm-up call.  Needs a CUDA device; there is no CPU fallback.
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
from chgnet_b200.phonons import Phonons  # noqa: E402
from oracle.phonons import PhononSpecKernels  # noqa: E402
from tools.time_phonons import gpu_card, timed  # noqa: E402
from tools.time_thermal_displacements import event_ms  # noqa: E402


def kernel_ms(ph: Phonons, mesh, omega_of, temps, repeats: int) -> float:
    """CUDA-event time of the chg_joint_dos calls of one joint_dos / phase_space call (its target chunks), on the
    frequencies that call uses; ``omega_of(nu) -> (targets, omega)``."""
    mesh, nu, _, tets, _, t = ph._jdos_mesh(mesh, temps)
    targets, omega = omega_of(nu)
    return event_ms(lambda: ph._joint_dos_chunks(mesh, nu, tets, targets, omega, t), repeats)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--jdos-mesh", type=int, default=20)
    ap.add_argument("--meshes", type=int, nargs="+", default=[8, 12, 16])
    ap.add_argument("--host-mesh", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_joint_dos.py needs a CUDA device")
    print(json.dumps({"card": gpu_card()}), flush=True)
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    ph = model.phonons(graphgen.limno2_structure(), [3, 3, 3], batch_size=a.batch_size)
    n3 = 3 * len(ph.p2s)
    n = a.jdos_mesh
    q = np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0], [0.25, 0.25, 0.0], [0.1, 0.2, 0.3]])
    q = np.round(q * n) / n
    for temps in (None, np.linspace(0.0, 1500.0, 31)):
        out, t_call = timed(lambda: ph.joint_dos((n,) * 3, q, temperatures=temps), a.repeats)

        def grid(nu):
            top = 2 * nu.max()
            om = torch.lerp(torch.zeros_like(top).expand(201), top.expand(201),
                            torch.arange(201, dtype=torch.float64, device="cuda") / 200)
            idx = np.round(q * n).astype(np.int64) % n
            tg = torch.as_tensor(((idx[:, 0] * n + idx[:, 1]) * n + idx[:, 2]).astype(np.int32)).cuda()
            return tg, om[None].expand(len(q), -1).contiguous()

        k_ms = kernel_ms(ph, (n,) * 3, grid, temps, a.repeats)
        print(json.dumps({"joint_dos_mesh": [n] * 3, "qpoints": len(q), "bands": n3, "frequency_points": 201,
                          "temperatures": 0 if temps is None else len(temps), "device_call_s": round(t_call, 4),
                          "device_joint_dos_kernel_ms_min": round(k_ms, 3), "n_imaginary": out["n_imaginary"],
                          "jdos_max": float(out["jdos"].max())}), flush=True)
    temps = [0.0, 300.0, 1000.0]
    device_out = {}
    for m in a.meshes:
        mesh = (m,) * 3
        out, t_call = timed(lambda: ph.phase_space(mesh, temps), a.repeats)
        device_out[m] = out
        k_ms = kernel_ms(ph, mesh, lambda nu: (torch.arange(nu.shape[0], dtype=torch.int32, device="cuda"), nu),
                         temps, a.repeats)
        items = m**3 * 6 * n3 * n3
        print(json.dumps({"phase_space_mesh": list(mesh), "targets": m**3, "bands": n3, "temperatures": len(temps),
                          "sorted_tetrahedra_per_slot": 2 * m**3 * items,
                          "device_call_s": round(t_call, 4), "device_joint_dos_kernel_ms_min": round(k_ms, 3),
                          "n_imaginary": out["n_imaginary"], "average_jdos": out["average_jdos"].tolist(),
                          "average_weighted_jdos": out["average_weighted_jdos"].tolist()}), flush=True)

    host = Phonons(ph.force_constants, ph.cell, device="cpu", kernels=PhononSpecKernels())
    hm = (a.host_mesh,) * 3
    dev = device_out.get(a.host_mesh) or ph.phase_space(hm, temps)
    t0 = time.perf_counter()
    ref = host.phase_space(hm, temps)
    t_host = time.perf_counter() - t0
    print(json.dumps({"host_mesh": list(hm), "host_spec_phase_space_s": round(t_host, 3),
                      "max_abs_jdos_diff_rel": float(np.abs(dev["jdos"] - ref["jdos"]).max() / np.abs(ref["jdos"]).max()),
                      "max_abs_weighted_diff_rel": float(np.abs(dev["weighted_jdos"] - ref["weighted_jdos"]).max()
                                                         / np.abs(ref["weighted_jdos"]).max()),
                      "n_imaginary_equal": dev["n_imaginary"] == ref["n_imaginary"]}), flush=True)


if __name__ == "__main__":
    main()
