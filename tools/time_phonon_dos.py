"""Time Phonons.dos and Phonons.group_velocities on the device against their fp64 specifications on the host.

    python tools/time_phonon_dos.py [--batch-size 16] [--repeats 3] [--mesh 40] [--gv-mesh 20] [--host-mesh 20]

With the force constants of LiMnO2 3x3x3 (0.3.0 weights): ``dos(projected=True)`` on a mesh^3 Gamma-centred mesh
(201 points), the ``chg_tetrahedron_dos`` kernel alone on the same frequencies and projections (CUDA events), and
``group_velocities`` on a gv-mesh^3 mesh.  Then the same calls with ``oracle/phonons.py``'s specifications on the
host (``Phonons(..., device="cpu", kernels=PhononSpecKernels())``), on a host-mesh^3 mesh, with the largest
difference from the device.  Prints the GPU name and power limit first: the times belong to that card.  Wall-clock
times are synchronised, the fastest of ``repeats`` after a warm-up call.  Needs a CUDA device; there is no CPU
fallback.
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
from chgnet_b200.phonons import Phonons, gamma_mesh, tetrahedra  # noqa: E402
from oracle.phonons import PhononSpecKernels  # noqa: E402
from tools.time_phonons import gpu_card, timed  # noqa: E402


def host_timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, time.perf_counter() - t0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--mesh", type=int, default=40)
    ap.add_argument("--gv-mesh", type=int, default=20)
    ap.add_argument("--host-mesh", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_phonon_dos.py needs a CUDA device")
    print(json.dumps({"card": gpu_card()}), flush=True)
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    ph = model.phonons(graphgen.limno2_structure(), [3, 3, 3], batch_size=a.batch_size)
    n_prim = len(ph.p2s)
    n3 = 3 * n_prim
    mesh = (a.mesh,) * 3
    out, t_dos = timed(lambda: ph.dos(mesh, projected=True), a.repeats)

    # the kernel alone, on the frequencies and projections dos() builds
    q = gamma_mesh(mesh)
    nu, proj = ph._mesh_frequencies(mesh, projected=True)
    omega = torch.as_tensor(out["frequency_points"]).cuda()
    tets = torch.as_tensor(tetrahedra(mesh, ph.cell.prim_lattice)).cuda()
    dos, idos = torch.empty_like(omega), torch.empty_like(omega)
    pdos = torch.empty(n_prim, len(omega), dtype=torch.float64, device="cuda")
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kernel_ms = []
    for _ in range(a.repeats + 1):
        start.record()
        ph.kernels.tetrahedron_dos(nu, mesh, tets, omega, dos, idos, proj, pdos)
        end.record()
        torch.cuda.synchronize()
        kernel_ms.append(start.elapsed_time(end))
    pairs = len(q) * 6 * n3
    print(json.dumps({"dos_mesh": list(mesh), "n_q": len(q), "modes": n3, "tetrahedron_band_pairs": pairs,
                      "frequency_points": len(omega), "projections": n_prim,
                      "device_dos_projected_s": round(t_dos, 4),
                      "device_tetrahedron_dos_kernel_ms_min": round(min(kernel_ms[1:]), 3),
                      "kernel_equals_dos_call": bool(np.array_equal(pdos.cpu().numpy(), out["projected_dos"])),
                      "integrated_dos_top": float(out["integrated_dos"][-1])}), flush=True)
    del nu, proj

    qg = gamma_mesh((a.gv_mesh,) * 3)
    v, t_gv = timed(lambda: ph.group_velocities(qg), a.repeats)
    print(json.dumps({"gv_mesh": [a.gv_mesh] * 3, "n_q": len(qg), "device_group_velocities_s": round(t_gv, 4),
                      "max_abs_v_THz_A": float(np.abs(v).max())}), flush=True)

    host = Phonons(ph.force_constants, ph.cell, device="cpu", kernels=PhononSpecKernels())
    hm = (a.host_mesh,) * 3
    dev_dos = ph.dos(hm, projected=True)
    host_dos, t_host_dos = host_timed(lambda: host.dos(hm, projected=True))
    qh = gamma_mesh(hm)
    dev_v = ph.group_velocities(qh)
    host_v, t_host_gv = host_timed(lambda: host.group_velocities(qh))
    print(json.dumps({"host_mesh": list(hm), "host_spec_dos_projected_s": round(t_host_dos, 3),
                      "host_spec_group_velocities_s": round(t_host_gv, 3),
                      "max_abs_dos_diff_rel": float(np.abs(dev_dos["projected_dos"] - host_dos["projected_dos"]).max()
                                                    / np.abs(host_dos["projected_dos"]).max()),
                      "max_abs_v_diff_rel": float(np.abs(dev_v - host_v).max() / np.abs(host_v).max())}), flush=True)


if __name__ == "__main__":
    main()
