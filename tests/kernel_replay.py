"""Record every kernel call of an engine run executed with the torch specifications on
the CPU, so that the same calls can be replayed through the CUDA library and compared
output by output (tests/test_kernels_gpu.py).  A recorded call keeps the argument layout
the engine used: strided column slices and aliased arguments replay as they ran."""
from __future__ import annotations

import torch

from oracle.kernel_specs import SpecKernels

# positional indices of the output arguments of each kernel method
OUT_ARGS = {
    "embed_atoms": [2],
    "edge_geometry": [6, 7, 8],
    "bond_basis_embed": [8, 9, 10, 11],
    "bond_basis_bwd": [11, 12],
    "angle_basis_embed": [5, 6],
    "angle_basis_bwd": [6, 7],
    "linear": [4],
    "gather_rows": [2],
    "scatter_rows": [2],
    "atom_conv_fwd": [9, 10, 11],
    "atom_conv_bwd": [10, 11, 12, 13],
    "segment_sum": [4],
    "atom_conv_fused": [10, 11],
    "bond_conv_fused": [11, 12, 13],
    "bond_conv_fwd": [10, 11, 12],
    "bond_conv_bwd": [8, 9, 10, 11, 12],
    "angle_update_fwd": [8, 9],
    "angle_update_bwd": [3, 4],
    "readout": [10, 11, 12, 13, 14],
    "magmom": [3],
    "force_virial": [10, 11],
    # training (trailing optional outputs above are training-only too)
    "wgrad": [2, 3],
    "colsum": [1],
    "readout_bwd": [7, 8, 9, 10, 11],
    "magmom_bwd": [4, 5],
    # second order
    "edge_tangent": [8, 9],
    "bond_basis_tangent": [9, 10, 11, 12],
    "bond_basis_bwd2": [12],
    "angle_basis_tangent": [6, 7],
    "angle_basis_bwd2": [7],
    "atom_conv_tan": [11, 12, 13],
    "atom_conv_bwd2": [13, 14, 15, 16],
    "bond_conv_tan": [12, 13, 14],
    "bond_conv_bwd2": [13, 14, 15, 16, 17],
    "angle_update_tan": [9, 10],
    "angle_update_bwd2": [5, 6],
    "readout_bwd2": [8, 9, 10, 11, 12, 13, 14, 15, 16],
}
SECOND_ORDER_KERNELS = {"edge_tangent", "bond_basis_tangent", "bond_basis_bwd2", "angle_basis_tangent", "angle_basis_bwd2",
                        "atom_conv_tan", "atom_conv_bwd2", "bond_conv_tan", "bond_conv_bwd2", "angle_update_tan",
                        "angle_update_bwd2", "readout_bwd2"}
# the unfused message kernels only run in training mode (they also save `pre`); inference uses the fused pair
TRAIN_KERNELS = {"wgrad", "colsum", "readout_bwd", "magmom_bwd", "atom_conv_fwd", "bond_conv_fwd"} | SECOND_ORDER_KERNELS
INFER_KERNELS = set(OUT_ARGS) - TRAIN_KERNELS


# a span starts on this byte boundary of its storage (the caching allocator's), so every argument rebuilt on a
# span keeps the address alignment the engine handed the kernel
ALIGN = 512


def extent(t: torch.Tensor) -> tuple[int, int]:
    """[lo, hi): the bytes of its storage a non-empty tensor touches, first to last element."""
    isz = t.element_size()
    lo = t.storage_offset() * isz
    return lo, lo + (1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))) * isz


def layout(args: list) -> tuple[list, dict[int, tuple[int, int]]]:
    """Group the non-empty tensor arguments of a call by storage.  Returns the spans ``(storage, lo, hi)``: per
    storage, the bytes from the first to the last element any argument touches (``lo`` rounded down to ALIGN), and
    ``where``: argument index -> (span index, byte offset of the argument's first element within its span)."""
    groups: dict[tuple, list[int]] = {}
    for i, a in enumerate(args):
        if isinstance(a, torch.Tensor) and a.numel():
            groups.setdefault((a.device, a.untyped_storage().data_ptr()), []).append(i)
    spans, where = [], {}
    for idx in groups.values():
        ext = [extent(args[i]) for i in idx]
        lo = min(e[0] for e in ext) // ALIGN * ALIGN
        for i, e in zip(idx, ext):
            where[i] = (len(spans), e[0] - lo)
        spans.append((args[idx[0]].untyped_storage(), lo, max(e[1] for e in ext)))
    return spans, where


def span_bytes(storage, lo: int, hi: int) -> torch.Tensor:
    """Bytes [lo, hi) of ``storage`` as a uint8 view."""
    return torch.empty(0, dtype=torch.uint8, device=storage.device).set_(storage, lo, (hi - lo,), (1,))


def rebuild(buf: torch.Tensor, offset: int, like: torch.Tensor, dtype: torch.dtype | None = None) -> torch.Tensor:
    """A view with the size and strides of ``like`` whose first element sits ``offset`` bytes into the uint8 tensor
    ``buf`` (``dtype``: reinterpret the bytes, same element size)."""
    dtype = dtype or like.dtype
    start = buf.storage_offset() + offset
    assert start % like.element_size() == 0, (start, like.dtype)
    return torch.empty(0, dtype=dtype, device=buf.device).set_(buf.untyped_storage(), start // like.element_size(),
                                                               like.shape, like.stride())


def snapshot(args: list) -> list:
    """The arguments of a call as the kernel sees them: each storage's touched span copied once, and each tensor
    argument a view of its span copy with its own offset, size and strides, so that column slices, leading
    dimensions and aliased arguments (``residual is y``) are kept.  Empty tensors are cloned; other values kept."""
    spans, where = layout(args)
    copies = [span_bytes(*s).clone() for s in spans]
    return [rebuild(copies[where[i][0]], where[i][1], a) if i in where
            else a.detach().clone() if isinstance(a, torch.Tensor) else a for i, a in enumerate(args)]


def record(calls: list, name: str, fn, args: tuple, out_args: list[int]) -> None:
    """Run ``fn(*args)`` and append ``(name, snapshot of the arguments before, outputs after)`` to ``calls``; the
    outputs (the fp32 specification's, the yardstick of fp32 arithmetic) are kept as contiguous copies."""
    snap = snapshot(list(args))
    fn(*args)
    outs = {i: args[i].detach().clone(memory_format=torch.contiguous_format) for i in out_args
            if i < len(args) and args[i] is not None}
    calls.append((name, snap, outs))


class RecordingKernels(SpecKernels):
    """Records every call of the kernels in ``recorded`` (kernel -> output argument indices); subclasses that mix in
    more specifications extend it."""

    recorded = OUT_ARGS

    def __init__(self) -> None:
        self.calls: list[tuple[str, list, dict[int, torch.Tensor]]] = []

    def __getattribute__(self, name):
        attr = super().__getattribute__(name)
        out_args = type(self).recorded.get(name)
        if out_args is not None and callable(attr):
            return lambda *args: record(self.calls, name, attr, args, out_args)
        return attr
