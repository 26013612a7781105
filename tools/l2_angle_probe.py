"""Times the angle-space kernels of a c3 step alone, L2 flushed before every launch as bench.py does, to see how much of
their time goes to gathers that miss L2.

For each kernel two index sets are timed on the same c3 graphs (batch 256 x 20-40 atoms, seeds 2000..):
  as-is        the real slot-j indices (`ang_js`): the j half of `pij` and the `wbg_s` / `g_agg` rows are read at random
  sequential   `ang_js` replaced by `ang_is`: every gathered table is read in angle order, so the random footprint is
               gone; the difference to as-is bounds what keeping the gathered tables resident in L2 can buy
plus the two gathered segment sums of the reverse angle scatter (g_pre over perm_js and perm_x) and their
unpermuted counterpart, and the AtomConv twins of the BondConv kernels.  Inputs are random (timings do not depend on
the values).

    python tools/l2_angle_probe.py [--iters 30] [--libs A.so,B.so,...] [--json OUT]

--libs times several builds of the kernel library in one process, interleaved launch by launch (default: this tree's
build).  Prints the GPU name and power limit, and one line per kernel and library: median and min of the per-launch
times in us."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

L2_FLUSH_BYTES = 256 << 20


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return f"nvidia-smi unavailable: {exc!r}"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--libs", default=None, help="comma-separated kernel libraries to compare (default: this tree's)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    from chgnet_b200 import graphgen
    from chgnet_b200 import _lib
    from chgnet_b200._lib import CudaKernels
    from chgnet_b200.batch import build_batch

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    K = CudaKernels(dev)
    libs = [os.path.abspath(p) for p in args.libs.split(",")] if args.libs else [_lib.LIB_PATH]
    handles = [_lib.load_library(p) for p in libs]
    b = build_batch(graphgen.random_graphs(256, 20, 40, 2000), dev, with_reverse=True)
    N, A, Es, Ed, Eu = b.n_atoms, b.n_angles, b.n_short, b.n_edges, b.n_bonds
    gen = torch.Generator(device=dev).manual_seed(0)

    def rnd(*shape, s=0.5):
        return torch.randn(*shape, device=dev, generator=gen) * s

    w2t, b2, w2 = rnd(64, 128, s=0.1), rnd(128, s=0.1), rnd(128, 64, s=0.1)
    ln = torch.cat([1.0 + rnd(64, s=0.1), rnd(64, s=0.1), 1.0 + rnd(64, s=0.1), rnd(64, s=0.1)]).contiguous()
    pij, px, pa, wbg_s = rnd(Es, 256), rnd(N, 128), rnd(A, 128), torch.rand(Es, 64, device=dev, generator=gen)
    ang, g_agg, g_ang = rnd(A, 64), rnd(Es, 64), rnd(A, 64)
    agg, s_pre, s_p = torch.empty(Es, 64, device=dev), torch.empty(A, 128, device=dev), torch.empty(A, 128, device=dev)
    ang_new, s_pa = torch.empty(A, 64, device=dev), torch.empty(A, 128, device=dev)
    g_pre, gw_i, gw_j = torch.empty(A, 128, device=dev), torch.empty(A, 64, device=dev), torch.empty(A, 64, device=dev)
    sp, spx = torch.empty(Es, 256, device=dev), torch.empty(N, 128, device=dev)
    pcn, pe, wag, g_x = rnd(N, 256), rnd(Eu, 128), torch.rand(Eu, 64, device=dev, generator=gen), rnd(N, 64)
    agg_x, a_p, a_gpre, a_gw = torch.empty(N, 64, device=dev), torch.empty(Ed, 128, device=dev), torch.empty(Ed, 128, device=dev), \
        torch.empty(Ed, 64, device=dev)
    fl_w = torch.empty(L2_FLUSH_BYTES // 4, device=dev)
    fl_r = torch.zeros(L2_FLUSH_BYTES // 4, device=dev)
    sink = torch.zeros((), device=dev)

    def flush():
        fl_w.zero_()
        sink.copy_(fl_r.sum())

    def time_us(fn) -> dict:
        """{library: times} of fn() with each library, the libraries taking turns launch by launch"""
        ts = {p: [] for p in libs}
        for it in range(3 + args.iters):
            for p, h in zip(libs, handles):
                K.lib = h
                flush()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                fn()
                e.record()
                e.synchronize()
                if it >= 3:
                    ts[p].append(s.elapsed_time(e) * 1e3)
        out = {}
        for p, t in ts.items():
            t.sort()
            out[os.path.relpath(p, ROOT)] = {"median_us": round(t[len(t) // 2], 1), "min_us": round(t[0], 1)}
        return out

    for h in handles:  # the reverse kernels read the saved rows: fill them once
        K.lib = h
        K.bond_conv_fused(pij, px, pa, wbg_s, b.ang_atom, b.ang_is, b.ang_js, b.ptr_is, w2t, b2, ln, agg, s_pre, s_p)
        K.atom_conv_fused(pcn, pe, wag, b.center, b.nbr, b.d2u, b.ptr_c, w2t, b2, ln, agg_x, a_p)
    torch.cuda.synchronize()
    res = {"gpu": gpu_info(), "tree": ROOT, "sizes": {"N": N, "A": A, "Es": Es, "Ed": Ed, "Eu": Eu},
           "table_MB": {"pij": Es * 1024 / 1e6, "wbg_s": Es * 256 / 1e6, "px": N * 512 / 1e6, "g_agg": Es * 256 / 1e6}}
    for label, js in (("as_is", b.ang_js), ("sequential", b.ang_is)):
        res[f"bond_conv_fused/{label}"] = time_us(lambda: K.bond_conv_fused(pij, px, pa, wbg_s, b.ang_atom, b.ang_is, js, b.ptr_is,
                                                                             w2t, b2, ln, agg, s_pre, s_p))
        res[f"bond_conv_bwd/{label}"] = time_us(lambda: K.bond_conv_bwd(s_pre, s_p, wbg_s, b.ang_is, js, g_agg, w2, ln, g_pre,
                                                                         gw_i, gw_j))
        res[f"angle_update_fwd/{label}"] = time_us(lambda: K.angle_update_fwd(pij, px, pa, ang, b.ang_atom, b.ang_is, js, ln,
                                                                               ang_new, s_pa))
    res["angle_update_bwd"] = time_us(lambda: K.angle_update_bwd(s_pa, g_ang, ln, g_pre))
    res["segment_sum/g_pre_by_is"] = time_us(lambda: K.segment_sum(g_pre, None, b.ptr_is, 0, sp[:, :128]))
    res["segment_sum/g_pre_by_js"] = time_us(lambda: K.segment_sum(g_pre, b.perm_js, b.ptr_js, 0, sp[:, 128:]))
    res["segment_sum/g_pre_by_x"] = time_us(lambda: K.segment_sum(g_pre, b.perm_x, b.ptr_x, 0, spx))
    res["atom_conv_fused"] = time_us(lambda: K.atom_conv_fused(pcn, pe, wag, b.center, b.nbr, b.d2u, b.ptr_c, w2t, b2, ln, agg_x, a_p))
    res["atom_conv_bwd"] = time_us(lambda: K.atom_conv_bwd(pcn, pe, wag, b.center, b.nbr, b.d2u, a_p, g_x, w2, ln, a_gpre, a_gw))
    for k, v in res.items():
        if isinstance(v, dict) and all(isinstance(x, dict) for x in v.values()):
            for lib, t in v.items():
                print(f"{k:34s} {t['median_us']:9.1f} us median {t['min_us']:9.1f} min   {lib}")
        else:
            print(f"{k}: {v}")
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
