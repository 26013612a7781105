"""Time the three-phonon path on the device by stage: third-order force constants, interaction strengths P, linewidths
and the RTA thermal conductivity.

    python tools/time_three_phonon.py [--batch-size 16] [--repeats 2] [--mesh 8] [--kappa-mesh 6] [--supercell 2]

With LiMnO2 on a supercell^3 supercell (0.3.0 weights): ``CHGNet.phonons(..., third_order=True)`` and the harmonic
part alone (wall clock, ending in a synchronise; their difference is the fc3 extraction); then on a mesh^3 mesh, for
one target q and every q1, ``chg_phonon_interaction`` and ``chg_imag_self_energy`` at 3 temperatures over the chunks
``Phonons.linewidths`` uses (CUDA events); ``Phonons.linewidths`` at that q and ``Phonons.thermal_conductivity`` on a
kappa-mesh^3 mesh (wall clock).  Prints the GPU name and power limit first: the times belong to that card.  Needs a
CUDA device; there is no CPU fallback.
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
from chgnet_b200.phonons import THERMAL_CUTOFF_THZ  # noqa: E402
from tools.time_phonons import gpu_card, timed  # noqa: E402
from tools.time_thermal_displacements import event_ms  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--mesh", type=int, default=8)
    ap.add_argument("--kappa-mesh", type=int, default=6)
    ap.add_argument("--supercell", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps({"gpu": gpu_card()}))
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"),
                             version="0.3.0").to("cuda")
    s = args.supercell
    st = graphgen.limno2_structure()
    t0 = time.perf_counter()
    ph = model.phonons(st, [s, s, s], batch_size=args.batch_size, third_order=True)
    torch.cuda.synchronize()
    t_all = time.perf_counter() - t0
    _, t_fc2 = timed(lambda: model.phonons(st, [s, s, s], batch_size=args.batch_size), 1)
    n = len(ph.cell.z)
    print(json.dumps({"supercell": [s] * 3, "atoms": n, "fc3_columns": 6 * len(ph.p2s) * 3 * n,
                      "phonons_third_order_s": t_all, "phonons_harmonic_s": t_fc2, "fc3_s": t_all - t_fc2}))

    m = (args.mesh,) * 3
    temps = torch.tensor([0.0, 300.0, 1000.0], dtype=torch.float64, device="cuda")
    mesh, nu, e, _, tets, _ = ph._three_phonon_mesh(m, None)
    n_mesh, nb = nu.shape
    target = n_mesh // 3 + 1
    chunk = ph._q1_chunk(len(temps))
    chunks = [torch.arange(a, min(a + chunk, n_mesh), dtype=torch.int32, device="cuda")
              for a in range(0, n_mesh, chunk)]
    ps = [ph._interactions(mesh, nu, e, target, q1) for q1 in chunks]
    gamma = torch.zeros(3, nb, dtype=torch.float64, device="cuda")
    omega = nu[target].contiguous()

    def interaction():
        for q1, p in zip(chunks, ps):
            ph.kernels.phonon_interaction(ph._fc3, ph._img_ptr, ph._img_vec, ph._s2p, ph._inv_sqrt_m,
                                          torch.as_tensor(ph.cell.prim_frac).cuda(), mesh, nu, e, target, q1,
                                          THERMAL_CUTOFF_THZ, p)

    def self_energy():
        for q1, p in zip(chunks, ps):
            ph.kernels.imag_self_energy(nu, mesh, tets, target, omega, q1, p, temps, THERMAL_CUTOFF_THZ, gamma)

    ms_p, ms_g = event_ms(interaction, args.repeats), event_ms(self_energy, args.repeats)
    q = np.unravel_index(target, m) / np.array(m)
    _, t_lw = timed(lambda: ph.linewidths(m, q, [0.0, 300.0, 1000.0]), args.repeats)
    print(json.dumps({"mesh": list(m), "bands": nb, "q1_per_call": chunk, "calls": len(chunks),
                      "chg_phonon_interaction_ms_per_target": ms_p, "chg_imag_self_energy_ms_per_target": ms_g,
                      "linewidths_one_q_s": t_lw}))
    km = (args.kappa_mesh,) * 3
    res, t_k = timed(lambda: ph.thermal_conductivity(km, [300.0]), 1)
    print(json.dumps({"kappa_mesh": list(km), "thermal_conductivity_s": t_k,
                      "kappa_300K_diag_W_per_mK": np.diag(res["kappa"][0]).tolist(),
                      "n_imaginary": res["n_imaginary"], "n_zero_linewidth": res["n_zero_linewidth"].tolist()}))


if __name__ == "__main__":
    main()
