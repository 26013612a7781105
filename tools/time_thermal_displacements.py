"""Time Phonons.thermal_displacement_matrices on the device against its fp64 specification on the host.

    python tools/time_thermal_displacements.py [--batch-size 16] [--repeats 3] [--meshes 20 40] [--host-mesh 20]

With the force constants of LiMnO2 3x3x3 (0.3.0 weights) and 31 temperatures from 0 to 1500 K:
``thermal_displacement_matrices`` on each mesh^3 Gamma-centred mesh (wall clock, ending in a synchronise), and, on the
same eigenvectors, the ``chg_thermal_displacements`` kernel alone and D(q) + ``torch.linalg.eigh`` alone (CUDA events
around the loop over the eigh chunks).  Then the same call with ``oracle/phonons.py``'s specification on
the host (``Phonons(..., device="cpu", kernels=PhononSpecKernels())``) on a host-mesh^3 mesh, with the
largest difference from the device.  Prints the GPU name and power limit first: the times belong to that card.  Times
are the fastest of ``repeats`` after a warm-up call.  Needs a CUDA device; there is no CPU fallback.
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
from chgnet_b200.phonons import DISPLACEMENT_A2_AMU_THZ, THERMAL_CUTOFF_THZ, Phonons, gamma_mesh  # noqa: E402
from chgnet_b200.phonons import _zero_gamma_acoustic  # noqa: E402
from oracle.phonons import PhononSpecKernels  # noqa: E402
from tools.time_phonons import gpu_card, timed  # noqa: E402


def event_ms(fn, repeats: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(repeats + 1):
        start.record()
        fn()
        end.record()
        torch.cuda.synchronize()
        ms.append(start.elapsed_time(end))
    return min(ms[1:])


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--meshes", type=int, nargs="+", default=[20, 40])
    ap.add_argument("--host-mesh", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_thermal_displacements.py needs a CUDA device")
    print(json.dumps({"card": gpu_card()}), flush=True)
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    ph = model.phonons(graphgen.limno2_structure(), [3, 3, 3], batch_size=a.batch_size)
    n_prim = len(ph.p2s)
    n3 = 3 * n_prim
    temps = np.linspace(0.0, 1500.0, 31)
    t_dev = torch.as_tensor(temps).cuda()
    device_out = {}
    for n in a.meshes:
        mesh = (n,) * 3
        out, t_call = timed(lambda: ph.thermal_displacement_matrices(mesh, temps), a.repeats)
        device_out[n] = out
        # the kernel alone, on the chunks of frequencies and eigenvectors the call builds (Gamma's three smallest |nu|
        # zeroed as there)
        q = gamma_mesh(mesh)
        chunks = []
        for s, nu, e in ph._eigh_chunks(q, eigenvectors=True, eigh_batch=ph.eigh_batch):
            if s.start == 0:
                _zero_gamma_acoustic(nu)
            chunks.append((nu, e.mT.contiguous()))
        acc = torch.zeros(len(temps), n_prim, 6, dtype=torch.float64, device="cuda")

        def kernels():
            acc.zero_()
            for nu, e in chunks:
                ph.kernels.thermal_displacements(nu, e, t_dev, THERMAL_CUTOFF_THZ, acc)

        kernel_ms = event_ms(kernels, a.repeats)
        eigh_ms = event_ms(lambda: list(ph._eigh_chunks(q, eigenvectors=True, eigh_batch=ph.eigh_batch)), a.repeats)
        v = acc.cpu().numpy() * (DISPLACEMENT_A2_AMU_THZ / len(q)) / ph.masses[None, :, None]
        same = bool(np.array_equal(v, out["cartesian"][..., [0, 1, 2, 1, 0, 0], [0, 1, 2, 2, 2, 1]]))
        del chunks
        print(json.dumps({"mesh": list(mesh), "n_q": len(q), "modes": n3, "temperatures": len(temps),
                          "eigh_chunks": -(-len(q) // ph.eigh_batch),
                          "device_call_s": round(t_call, 4),
                          "device_thermal_displacements_kernel_ms_min": round(kernel_ms, 3),
                          "device_dynamical_matrices_plus_eigh_ms_min": round(eigh_ms, 3),
                          "n_imaginary": out["n_imaginary"],
                          "U_300K_diag_A2": np.diagonal(out["cartesian"][6], axis1=1, axis2=2).round(6).tolist(),
                          "kernel_loop_equals_call": same}), flush=True)

    host = Phonons(ph.force_constants, ph.cell, device="cpu", kernels=PhononSpecKernels())
    hm = (a.host_mesh,) * 3
    dev = device_out.get(a.host_mesh) or ph.thermal_displacement_matrices(hm, temps)
    t0 = time.perf_counter()
    ref = host.thermal_displacement_matrices(hm, temps)
    t_host = time.perf_counter() - t0
    print(json.dumps({"host_mesh": list(hm), "host_spec_s": round(t_host, 3),
                      "max_abs_U_diff_rel": float(np.abs(dev["cartesian"] - ref["cartesian"]).max()
                                                  / np.abs(ref["cartesian"]).max()),
                      "max_abs_cif_diff_rel": float(np.abs(dev["cif"] - ref["cif"]).max() / np.abs(ref["cif"]).max()),
                      "n_imaginary_equal": dev["n_imaginary"] == ref["n_imaginary"]}), flush=True)


if __name__ == "__main__":
    main()
