"""Time ``CHGNet.effective_phonons`` on the device, stage by stage.

    python tools/time_effective_phonons.py [--supercells 2 3] [--samples 256] [--iterations 2] [--batch-size 16]

LiMnO2 on supercell^3 supercells (0.3.0 weights) at 300 K, quantum: per iteration the time of the sampler
(``chg_sample_displacements``), the engine (the replica forces), the moments (``chg_displacement_moments``) and
the rest of the iteration (eigendecompositions and the fit), from CUDA events, with the exact per-sample graphs of the
product path (``structures_to_batch``); and for the alternative, one shared graph of the reference positions with both
cutoffs widened by a skin of 2 max |u| (rounded up to 0.05 A), the skin the iteration's samples need, the angle counts
with and without it, and the engine time of the same samples through it (or the out-of-memory error it meets).
Prints the GPU name and power limit first: the times belong to that card.  Needs a CUDA device; there is no CPU fallback.
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
from chgnet_b200.batch import build_batch  # noqa: E402
from chgnet_b200.model import CHGNet, GraphConverter, _ReplicaForces  # noqa: E402
from chgnet_b200.phonons import effective_force_constants, make_supercell  # noqa: E402
from tools.time_phonons import gpu_card  # noqa: E402


class _Timer:
    """Accumulates CUDA-event times (ms) per stage name."""

    def __init__(self):
        self.pending, self.ms = [], {}

    def wrap(self, name, fn):
        def run(*a, **kw):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            out = fn(*a, **kw)
            end.record()
            self.pending.append((name, start, end))
            return out
        return run

    def collect(self):
        torch.cuda.synchronize()
        for name, s, e in self.pending:
            self.ms[name] = self.ms.get(name, 0.0) + s.elapsed_time(e)
        self.pending = []
        out, self.ms = self.ms, {}
        return out


class _Kernels:
    def __init__(self, kernels, timer):
        self.sample_displacements = timer.wrap("sampler", kernels.sample_displacements)
        self.displacement_moments = timer.wrap("moments", kernels.displacement_moments)


def _skin_graph(model, sc, skin):
    gc = model.graph_converter
    return GraphConverter(gc.atom_graph_cutoff + skin, gc.bond_graph_cutoff + skin)((sc.z, sc.frac, sc.lattice))


def _angles(g):
    return int(g.bond_graph.shape[0]) if g.bond_graph.dim() == 2 else 0


def _skinned_engine_ms(model, sc, graph, chunks):
    """Engine time (ms, host clock around synchronised calls) of the sample chunks through copies of ``graph``."""
    nat, batches, total = model._get_native(), {}, 0.0
    for f in chunks:
        m = f.shape[0]
        if m not in batches:
            batches[m] = build_batch([graph] * m, model.device, with_reverse=True,
                                     compact_bonds=not model._arch.get("mlp_out_bias", False))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batches[m].frac.copy_(f.reshape(-1, 3))
        nat(batches[m], need_grad=True)
        torch.cuda.synchronize()
        total += (time.perf_counter() - t0) * 1e3
    return total


def run(model, n, samples, iterations, batch_size):
    from chgnet_b200._lib import CudaKernels

    s = graphgen.limno2_structure()
    sc = make_supercell(*s, [n, n, n])
    harm = model.phonons(s, [n, n, n], batch_size=batch_size)
    timer = _Timer()
    reps = _ReplicaForces(model, sc)
    ref = torch.as_tensor(np.asarray(sc.frac, dtype=np.float32)).cuda().double()
    lat = torch.as_tensor(np.ascontiguousarray(sc.lattice)).cuda()
    seen = []

    def forces(frac):
        seen.append(frac.clone())
        return reps(frac)

    kern = _Kernels(CudaKernels("cuda"), timer)
    rows = []
    for it in range(iterations):
        seen.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        # one iteration per call, seeded per iteration
        _, info = effective_force_constants(timer.wrap("engine", forces), sc, harm.force_constants, 300.0,
                                            kernels=kern, device="cuda", n_samples=samples, n_iterations=1,
                                            seed=it, batch_size=batch_size)
        torch.cuda.synchronize()
        total = (time.perf_counter() - t0) * 1e3
        ms = timer.collect()
        ms["total"] = total
        ms["solve_and_rest"] = total - ms["sampler"] - ms["engine"] - ms["moments"]
        chunks = seen[1:]
        u_max = max(float(((f - ref[None]) @ lat).norm(dim=-1).max()) for f in chunks)
        skin = float(np.ceil(2 * u_max / 0.05 - 1e-9) * 0.05)
        row = {"iteration": it, "ms": {k: round(v, 2) for k, v in ms.items()}, "max_u_A": u_max, "skin_A": skin,
               "sigma_a": info["sigma_a"], "n_imaginary": info["history"][0]["n_imaginary"]}
        g = _skin_graph(model, sc, skin)
        row["angles_no_skin"], row["angles_skin"] = _angles(_skin_graph(model, sc, 0.0)), _angles(g)
        try:
            row["engine_skinned_ms"] = round(_skinned_engine_ms(model, sc, g, chunks), 2)
        except (torch.OutOfMemoryError, RuntimeError) as e:  # the skinned batch may not fit
            row["engine_skinned_ms"] = f"out of memory: {str(e)[:90]}"
        torch.cuda.empty_cache()
        rows.append(row)
    return {"supercell": n, "atoms": len(sc.z), "samples": samples, "batch_size": batch_size, "iterations": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--supercells", type=int, nargs="+", default=[2, 3])
    ap.add_argument("--samples", type=int, default=256)
    ap.add_argument("--iterations", type=int, default=2)
    ap.add_argument("--batch-size", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_effective_phonons needs a CUDA device")
    print(json.dumps({"card": gpu_card()}))
    model = CHGNet.from_file(os.path.join(ROOT, "tests", "golden", "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")
    for n in args.supercells:
        print(json.dumps(run(model, n, args.samples, args.iterations, args.batch_size)), flush=True)
    print(json.dumps({"card_after": gpu_card()}))


if __name__ == "__main__":
    main()
