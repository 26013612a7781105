"""Check recorded kernel calls against an fp64 evaluation of their torch specifications.

A recorded call is ``(name, snapshot, outs)`` (``tests/kernel_replay.py``): the kernel's arguments as the engine
handed them in, and the outputs the fp32 specification wrote.  For each call:

* ``reference64`` runs the specification (``oracle.elastic.ElasticSpecKernels``, which includes the Hessian and
  training kernels) on the same snapshot with float32 tensors promoted to float64, integer and float64 tensors
  cloned and scalars unchanged: the fp64 reference ``ref`` for the very fp32 inputs the kernel sees.  The recorded
  fp32 outputs give the yardstick ``e32 = max|spec32 - ref|`` of what fp32 arithmetic costs on that output.
* ``replay`` runs the CUDA kernel on the same snapshot in the engine's layout (``place``: each storage span between
  two NaN guard bands, every argument a view with its recorded offset and strides, aliasing kept), with every output
  the kernel must overwrite filled with NaN first (an output row or tail the kernel forgets to write then fails
  instead of matching stale values); outputs the header documents as accumulated (``+=``) and outputs that share
  elements with an input (``residual is y``) keep their recorded contents.  After the call both guard bands and every
  span byte outside the declared outputs must be bitwise unchanged: a write past a ragged last tile, into the unused
  columns of a strided output, into rows a row scatter does not own, or into an input is a stray write.
* ``Checker.check`` applies the rule per call and output: with ``scale = max|ref|``,
  ``max|out - ref| <= max(R * scale, K * e32)``; an output whose reference is all zero must be exactly zero, and a
  NaN or Inf fails.  ``Checker.table`` prints the worst ``err / scale`` and ``err / tol`` of every kernel output.
"""
from __future__ import annotations

import torch

from kernel_replay import OUT_ARGS, extent, layout, rebuild, span_bytes
from oracle.elastic import ElasticSpecKernels

# bytes of guard band before and after each replayed span (more than one 128-row tile of 256-column fp32 rows, 128 KiB),
# filled with 0xff: a NaN in fp32 and fp64, -1 in the index types
GUARD = 1 << 20
NAN_BYTE = 0xFF
_SAME_SIZE_INT = {1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}

# relative floor and multiple of the fp32 specification's own error.  Calibrated on one NVIDIA H100 80GB HBM3 (400 W
# power limit) over tests/test_kernels_fp64_gpu.py and the per-kernel replays of test_kernels_gpu / test_hessian_gpu /
# test_elastic_gpu: outside the overrides below the worst output sits at 0.42 of its tolerance (bond_conv_bwd g_pre),
# most below 0.3; many sit at exactly 0.25, i.e. the kernel's error equals the fp32 specification's.
R = 4e-6
K = 4.0
# per-output (R, K), (kernel, output argument) -> dict(r=..., k=...), each with its reason and the H100 figure that set it
OVERRIDES: dict[tuple[str, int], dict] = {
    # dW of chg_wgrad's tensor-core kernel: 3xTF32 products summed in fp32 per CTA over thousands of rows (the per-CTA
    # partials are then summed in fp64); at the 64k-row reductions of a production training step the worst error is
    # 6.0e-6 of max|dW| while the fp32 specification's (blocked) sum stays below 1e-6.  The error grows with the rows
    # each CTA sums: over the 223k angle rows of the high-coordination batch (~845 rows per CTA) it is 1.78e-5
    ("wgrad", 2): dict(r=4e-5),
    # chg_linear's 3xTF32 wgmma kernels on the adjoint rows of the strain second-derivative pass (8 x 144-atom cells):
    # 3.9e-6 of scale, against an fp32 specification 30x closer; everywhere else below 3e-6
    ("linear", 4): dict(r=8e-6),
    # theta = acos(u) is ill-conditioned near collinear bond pairs (|dtheta/du| up to 1/sqrt(2e-6) = 707 with the
    # (1 - 1e-6) clamp), so the per-element difference of two fp32 roundings of u (kernel vs specification) is amplified
    # there by up to that factor; the kernel's worst element need not be the specification's worst.  H100: 7.7 x e32
    # for g_rhat (6.7e-5 of scale) and 4.4 x e32 for a0 (4.5e-6 of scale) on the 0.2.0-shaped random cells
    ("angle_basis_bwd", 6): dict(k=16.0),
    ("angle_basis_embed", 5): dict(k=8.0),
}

# output arguments of the Hessian-vector and strain second-derivative kernels (the others are in OUT_ARGS)
SECOND_DERIV_OUT_ARGS = {"bond_basis_hvp": [12], "angle_basis_hvp": [7], "edge_tangent_bwd": [10],
                         "edge_tangent_bwd_virial": [12, 13]}
ALL_OUT_ARGS = {**OUT_ARGS, **SECOND_DERIV_OUT_ARGS}
# outputs the kernels accumulate into (include/chgnet_b200.h: g_rhat, g_freq, g_ln, e_graph / e_ref, force, virial,
# chg_colsum's out, magmom_bwd's g_x and the second-order accumulators); every other output is overwritten
ACCUMULATED = {
    "bond_basis_bwd": {12}, "angle_basis_bwd": {6, 7}, "atom_conv_bwd": {13}, "bond_conv_bwd": {12},
    "angle_update_bwd": {4}, "readout": {12, 13}, "force_virial": {10, 11}, "colsum": {1}, "magmom_bwd": {4},
    "bond_basis_bwd2": {12}, "angle_basis_bwd2": {7}, "atom_conv_bwd2": {16}, "bond_conv_bwd2": {17},
    "angle_update_bwd2": {6}, "bond_basis_hvp": {12}, "angle_basis_hvp": {7}, "edge_tangent_bwd": {10},
    "edge_tangent_bwd_virial": {12, 13},
}

_SPEC = ElasticSpecKernels()


def _promote(a):
    if isinstance(a, torch.Tensor):
        return a.double() if a.dtype == torch.float32 else a.clone()
    return a


def reference64(name: str, snap: list) -> dict[int, torch.Tensor]:
    """fp64 outputs of the specification of kernel ``name`` on the fp32 inputs of ``snap``."""
    args = [_promote(a) for a in snap]
    getattr(_SPEC, name)(*args)
    return {i: args[i] for i in ALL_OUT_ARGS[name] if i < len(args) and args[i] is not None}


def _rows(name: str, args: list, i: int):
    """The rows of output ``i`` the kernel writes (``None``: all of them)."""
    if name == "linear" and i == 4:
        return args[6]  # y_rows
    if name == "scatter_rows" and i == 2:
        return args[1]
    return None


def poison(name: str, args: list, keep: set[int] = frozenset()) -> None:
    """NaN into every output of the call that the kernel must write (the rows it writes, for row scatters).
    ``keep``: outputs that share elements with an input (``residual is y``) keep their contents."""
    nan = float("nan")
    for i in ALL_OUT_ARGS[name]:
        t = args[i] if i < len(args) else None
        if t is None or i in ACCUMULATED.get(name, ()) or i in keep:
            continue
        if name == "segment_sum" and args[3]:
            continue  # accumulate = 1
        if name == "readout_bwd" and i == 11 and args[1] is None:
            continue  # xhat: only with a LayerNorm
        if name == "readout_bwd2" and i in (15, 16) and args[2] is None:
            continue
        if name == "linear" and args[6] is not None:
            t[args[6].long()] = nan  # y_rows: the other rows keep their contents
        elif name == "scatter_rows":
            t[args[1].long()] = nan
        else:
            t.fill_(nan)


class Checker:
    """The rule, applied output by output, with the worst margins kept per (kernel, output)."""

    def __init__(self, r: float = R, k: float = K, overrides: dict | None = None) -> None:
        self.r, self.k = r, k
        self.overrides = OVERRIDES if overrides is None else overrides
        self.worst: dict[tuple[str, int], list] = {}  # -> [err/scale, err/tol, calls]
        self.strays: dict[str, list] = {}  # kernel -> [first stray write, calls with one]
        self.failures: list[str] = []

    def stray(self, name: str, where: str) -> None:
        """A write of kernel ``name`` outside its declared outputs (``where``: the bytes written)."""
        s = self.strays.setdefault(name, [where, 0])
        s[1] += 1
        self.failures.append(f"{name} stray write: {where}")

    def check(self, name: str, idx: int, got: torch.Tensor, ref: torch.Tensor, spec32: torch.Tensor) -> bool:
        got = got.detach().double().cpu()
        if ref.numel() == 0:
            return True
        e32 = float((spec32.double() - ref).abs().max())
        scale = float(ref.abs().max())
        finite = bool(torch.isfinite(got).all())
        err = float((got - ref).abs().max()) if finite else float("inf")
        o = self.overrides.get((name, idx), {})
        tol = max(o.get("r", self.r) * scale, o.get("k", self.k) * e32)
        ok = finite and (err == 0.0 if scale == 0.0 else err <= tol)
        w = self.worst.setdefault((name, idx), [0.0, 0.0, 0])
        w[0] = max(w[0], err / scale if scale else (0.0 if err == 0.0 else float("inf")))
        w[1] = max(w[1], err / tol if tol else (0.0 if err == 0.0 else float("inf")))
        w[2] += 1
        if not ok:
            self.failures.append(f"{name} out[{idx}]: max err {err:.3e} > tol {tol:.3e} "
                                 f"(scale {scale:.3e}, fp32 spec err {e32:.3e}, finite {finite})")
        return ok

    def check_call(self, name: str, args: list, ref: dict, outs: dict) -> None:
        for idx, want in ref.items():
            self.check(name, idx, args[idx], want, outs[idx])

    @property
    def kernels(self) -> set[str]:
        return {n for n, _ in self.worst}

    def table(self, title: str = "") -> str:
        lines = [f"margins {title}: kernel out[arg]  worst err/scale  worst err/tol  calls"]
        for (n, i), (es, et, c) in sorted(self.worst.items()):
            lines.append(f"  {n:24s} out[{i:2d}]  {es:9.2e}  {et:6.3f}  {c}")
        for n, (where, c) in sorted(self.strays.items()):
            lines.append(f"  {n:24s} stray     {where}  {c}")
        return "\n".join(lines)

    def assert_ok(self, title: str = "") -> None:
        print(self.table(title))
        assert not self.failures, f"{len(self.failures)} outputs fail the fp64 rule:\n" + "\n".join(self.failures[:40])


class StreamedCalls(list):
    """Drop-in for a recorder's ``calls`` list that replays and checks each call as it is recorded and keeps none of
    them (a production-size training step records tens of GB of snapshots)."""

    def __init__(self, cuda_kernels, checker: Checker) -> None:
        super().__init__()
        self.cuda_kernels, self.checker = cuda_kernels, checker

    def append(self, call) -> None:
        replay([call], self.cuda_kernels, self.checker)


def place(snap: list, device="cuda") -> tuple[list, list, list]:
    """The arguments of a recorded call on ``device``, in the layout the engine handed the kernel: each span of the
    snapshot (``kernel_replay.layout``) in its own buffer between two GUARD-byte bands of NAN_BYTE, every tensor
    argument rebuilt on it with its recorded offset, size and strides (so views and aliasing are as recorded).
    Returns ``(args, buffers, where)``; span ``s`` starts GUARD bytes into ``buffers[s]``."""
    spans, where = layout(snap)
    bufs = []
    for storage, lo, hi in spans:
        n = hi - lo
        buf = torch.full((GUARD + n + GUARD,), NAN_BYTE, dtype=torch.uint8, device=device)
        buf[GUARD : GUARD + n].copy_(span_bytes(storage, lo, hi))
        bufs.append(buf)
    args = [rebuild(bufs[where[i][0]], GUARD + where[i][1], a) if i in where
            else a.detach().clone().to(device) if isinstance(a, torch.Tensor) else a for i, a in enumerate(snap)]
    return args, bufs, where


def _mask_view(masks: list, where: dict, args: list, i: int, rows=None) -> torch.Tensor:
    """The bytes of argument ``i`` (only ``rows``, when given) in its span's byte mask, one integer per element."""
    s, off = where[i]
    v = rebuild(masks[s], GUARD + off, args[i], _SAME_SIZE_INT[args[i].element_size()])
    return v if rows is None else v[rows.long()]


def _cover(masks: list, where: dict, args: list, i: int, rows=None) -> None:
    s, off = where[i]
    v = rebuild(masks[s], GUARD + off, args[i], _SAME_SIZE_INT[args[i].element_size()])
    if rows is None:
        v.fill_(-1)  # every byte 0xff
    else:
        v[rows.long()] = -1


def replay(calls, cuda_kernels, checker: Checker, refs: list | None = None, device="cuda") -> None:
    """Run every recorded call through ``cuda_kernels`` (``chgnet_b200._lib.CudaKernels``) on arguments placed by
    ``place`` and check it: both guard bands and every span byte outside the declared outputs (ALL_OUT_ARGS, only
    the rows written for the row scatters) bitwise unchanged, and the outputs against fp64 (``Checker.check``).
    ``refs``: the ``reference64`` of each call when already computed (a cached recording replayed more than once)."""
    for k, (name, snap, outs) in enumerate(calls):
        ref = refs[k] if refs is not None else reference64(name, snap)
        args, bufs, where = place(snap, device)
        out_idx = [i for i in ALL_OUT_ARGS[name] if i in where]
        declared = [torch.zeros_like(b) for b in bufs]
        inputs = [torch.zeros_like(b) for b in bufs]
        for i in where:
            if i not in out_idx:
                _cover(inputs, where, args, i)
        for i in out_idx:
            _cover(declared, where, args, i, _rows(name, args, i))
        keep = {i for i in out_idx if bool(_mask_view(inputs, where, args, i, _rows(name, args, i)).any())}
        poison(name, args, keep)
        before = [b.clone() for b in bufs]
        getattr(cuda_kernels, name)(*args)
        if torch.device(device).type == "cuda":
            torch.cuda.synchronize()
        for s, (buf, old, mask) in enumerate(zip(bufs, before, declared)):
            stray = torch.nonzero((buf != old) & (mask == 0)).flatten()
            if stray.numel():
                checker.stray(name, _describe(int(stray[0]), int(stray[-1]) + 1, s, buf.numel(), where, snap))
        checker.check_call(name, args, ref, outs)


def _describe(a: int, b: int, s: int, size: int, where: dict, snap: list) -> str:
    """Byte range [a, b) of the buffer of span ``s``, relative to the span's start, and what it lies in."""
    first = a - GUARD
    args = [i for i, (t, off) in where.items()
            if t == s and off <= first < off + extent(snap[i])[1] - extent(snap[i])[0]]
    parts = [p for p, hit in (("front guard", a < GUARD), ("back guard", b > size - GUARD),
                              (f"first in the bytes of args {args}", bool(args))) if hit]
    return f"bytes [{first}, {b - GUARD}) of span {s} ({', '.join(parts) or 'between arguments'})"
