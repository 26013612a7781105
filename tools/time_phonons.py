"""Time CHGNet.phonons: compact force constants against predict_hessian of the supercell, and frequencies on a mesh on
the device against the fp64 specification of the dynamical matrices on the host.

    python tools/time_phonons.py [--batch-size 16] [--repeats 2] [--mesh 20]

For LiMnO2 3x3x3 and 4x4x4 (0.3.0 weights): ``CHGNet.phonons`` (supercell graph + 3 n_prim = 24 Hessian-vector
products) against ``predict_hessian`` of the same supercell (3N products), and max|Phi - p2s rows of H|.  Then, with
the 3x3x3 force constants, ``Phonons.frequencies`` on a mesh^3 Gamma-centred mesh on the device (the
``chg_dynamical_matrices`` kernel alone timed with CUDA events, and the whole call with eigh and copies) against
``oracle/phonons.py``'s specification of D(q) plus ``numpy.linalg.eigvalsh`` on the host.  Prints the GPU name and power
limit first: the times belong to that card.  Wall-clock times are synchronised, the fastest of ``repeats`` after a
warm-up call.  Needs a CUDA device; there is no CPU fallback.
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
from chgnet_b200.phonons import THZ_PER_SQRT_EV_A2_AMU, Phonons, gamma_mesh  # noqa: E402
from oracle.phonons import PhononSpecKernels  # noqa: E402


def gpu_card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[:1]}


def timed(fn, repeats: int):
    out = fn()  # warm-up: module loads, allocator, batch shapes
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return out, min(times)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--mesh", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_phonons.py needs a CUDA device")
    print(json.dumps({"card": gpu_card()}), flush=True)
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    prim = graphgen.limno2_structure()
    keep = None
    for s in (3, 4):
        ph, t_fc = timed(lambda: model.phonons(prim, [s, s, s], batch_size=a.batch_size), a.repeats)
        sc = ph.cell
        n = len(sc.z)
        h, t_h = timed(lambda: model.predict_hessian((sc.z, sc.frac, sc.lattice), batch_size=a.batch_size), a.repeats)
        rows = h.reshape(n, 3, n, 3)[sc.p2s].transpose(0, 2, 1, 3)
        print(json.dumps({"cell": f"LiMnO2 {s}x{s}x{s}", "n_atoms": n, "batch_size": a.batch_size,
                          "phonons_fc_s": round(t_fc, 4), "fc_columns": 3 * len(sc.p2s),
                          "predict_hessian_s": round(t_h, 4), "hessian_columns": 3 * n,
                          "max_abs_fc_minus_hessian_rows": float(np.abs(ph.force_constants - rows).max()),
                          "max_abs_fc": float(np.abs(ph.force_constants).max())}), flush=True)
        if s == 3:
            keep = ph
        del h
    ph = keep
    q = gamma_mesh((a.mesh,) * 3)
    nu, t_dev = timed(lambda: ph.frequencies(q), a.repeats)
    qd = torch.as_tensor(q).cuda()
    n3 = 3 * len(ph.p2s)
    d = torch.empty(len(q), n3, n3, dtype=torch.complex128, device="cuda")
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    kernel_ms = []
    for _ in range(a.repeats + 1):
        start.record()
        ph.kernels.dynamical_matrices(ph._fc, ph._img_ptr, ph._img_vec, ph._s2p, ph._inv_sqrt_m, qd, d)
        end.record()
        torch.cuda.synchronize()
        kernel_ms.append(start.elapsed_time(end))
    host = Phonons(ph.force_constants, ph.cell, device="cpu", kernels=PhononSpecKernels())
    t0 = time.perf_counter()
    lam = np.linalg.eigvalsh(host.dynamical_matrices(q).numpy())
    t_host = time.perf_counter() - t0
    nu_host = np.sign(lam) * np.sqrt(np.abs(lam)) * THZ_PER_SQRT_EV_A2_AMU
    lam_dev = np.sign(nu) * (nu / THZ_PER_SQRT_EV_A2_AMU) ** 2
    print(json.dumps({"mesh": [a.mesh] * 3, "n_q": len(q), "modes": n3,
                      "device_frequencies_s": round(t_dev, 4), "device_kernel_ms_min": round(min(kernel_ms[1:]), 3),
                      "host_spec_plus_eigvalsh_s": round(t_host, 3),
                      "max_abs_eigenvalue_diff_rel": float(np.abs(lam_dev - lam).max() / np.abs(lam).max()),
                      "max_abs_nu_diff_THz": float(np.abs(nu - nu_host).max()),
                      "min_nu_THz": float(nu.min()), "max_nu_THz": float(nu.max())}), flush=True)


if __name__ == "__main__":
    main()
