"""ctypes binding of ``libchgnet_b200.so`` (the C ABI in include/chgnet_b200.h).

PyTorch is plumbing here: tensors only provide device memory (``data_ptr()``) and
the current CUDA stream.  There is NO fallback: if the shared library is missing
or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int32, c_int64, c_void_p

import torch
from torch import Tensor

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libchgnet_b200.so")

P, I, F, D, I64 = c_void_p, c_int32, c_float, c_double, c_int64

# name -> argument ctypes (the trailing stream pointer included); mirrors the header 1:1
SIGNATURES: dict[str, list] = {
    "chg_embed_atoms": [P, P, I, P, P],
    "chg_edge_geometry": [P, P, P, P, P, P, I, P, P, P, P],
    "chg_bond_basis_embed": [P, P, I, P, P, I, F, F, I, P, P, P, P, P, P],
    "chg_bond_basis_bwd": [P, P, I, P, P, I, F, F, I, P, P, P, P, P, P, P],
    "chg_angle_basis_embed": [P, P, P, I, P, I, P, P, P, P],
    "chg_angle_basis_bwd": [P, P, P, I, P, I, P, P, P, P, P],
    "chg_linear": [P, P, I, I, P, P, P, P, I, P, P],
    "chg_gather_rows": [P, P, I, I, P, P],
    "chg_scatter_rows": [P, P, I, I, P, P],
    "chg_atom_conv_fwd": [P, P, P, P, P, P, I, P, P, P, P, P, P, P],
    "chg_atom_conv_bwd": [P, P, P, P, P, P, I, P, P, P, P, P, P, P, P, P],
    "chg_segment_sum": [P, I, P, P, I, I, I, P, I, P],
    "chg_atom_conv_fused": [P, P, P, P, P, P, P, I, I, P, P, P, P, P, P, P],
    "chg_bond_conv_fused": [P, P, P, P, P, P, P, P, I, I, P, P, P, P, P, P, P, P],
    "chg_bond_conv_fwd": [P, P, P, P, P, P, P, I, P, P, P, P, P, P, P],
    "chg_bond_conv_bwd": [P, P, P, P, P, I, P, P, P, P, P, P, P, P, P],
    "chg_angle_update_fwd": [P, P, P, P, P, P, P, I, P, P, P, P],
    "chg_angle_update_bwd": [P, P, I, P, P, P, P],
    "chg_readout": [P, P, P, I, P, P, P, P, I, P, F, P, P, P, P, P, P, P],
    "chg_magmom": [P, I, P, F, P, P],
    "chg_force_virial": [P, P, P, P, P, P, P, P, P, P, I, P, P, P],
    # training
    "chg_wgrad": [P, P, I, P, I, P, I, P, I, I, P, I, P, P, P],
    "chg_colsum": [P, I, P, I, P, I, I, P, P],
    "chg_readout_bwd": [P, I, P, P, P, P, I, P, P, P, P, P, P, P, P],
    "chg_magmom_bwd": [P, I, P, F, P, P, P, P],
    "chg_loss_terms": [P, P, I, I, F, P, P, P],
    "chg_adam_step": [P, P, P, P, I64, F, F, F, F, F, I, P],
    # second order (force / stress losses)
    "chg_edge_tangent": [P, P, P, P, P, P, P, P, I, P, P, P],
    "chg_bond_basis_tangent": [P, P, P, I, P, P, I, F, F, I, P, P, P, P, P, P],
    "chg_bond_basis_bwd2": [P, P, P, I, P, P, I, F, F, I, P, P, P, P, P, P],
    "chg_angle_basis_tangent": [P, P, P, P, I, P, I, P, P, P, P],
    "chg_angle_basis_bwd2": [P, P, P, P, I, P, I, P, P, P, P],
    "chg_atom_conv_tan": [P, P, P, P, P, P, P, I, P, P, P, P, P, P, P, P],
    "chg_atom_conv_bwd2": [P, P, P, P, P, P, P, P, P, I, P, P, P, P, P, P, P, P, P],
    "chg_bond_conv_tan": [P, P, P, P, P, P, P, P, I, P, P, P, P, P, P, P, P],
    "chg_bond_conv_bwd2": [P, P, P, P, P, P, P, P, P, I, P, P, P, P, P, P, P, P, P, P],
    "chg_angle_update_tan": [P, P, P, P, P, P, P, I, P, P, P, P, P],
    "chg_angle_update_bwd2": [P, P, P, P, I, P, P, P, P],
    "chg_readout_bwd2": [P, P, I, P, P, P, P, I, P, P, P, P, P, P, P, P, P, P, P, P],
    # Hessian-vector products
    "chg_bond_basis_hvp": [P, P, P, I, P, P, I, F, F, I, P, P, P, P, P, P],
    "chg_angle_basis_hvp": [P, P, P, P, I, P, I, P, P, P, P],
    "chg_edge_tangent_bwd": [P, P, P, P, P, P, P, P, P, P, I, P, P],
    "chg_edge_tangent_bwd_virial": [P, P, P, P, P, P, P, P, P, P, P, P, I, P, P, P],
    # phonons
    "chg_dynamical_matrices": [P, P, P, P, P, I, I, P, I, P, P],
    "chg_dynamical_matrix_derivatives": [P, P, P, P, P, I, I, P, I, P, P, P],
    "chg_tetrahedron_dos": [P, I, I, I, I, P, P, I, P, I, P, P, P, P, P],
    "chg_thermal_displacements": [P, P, I, I, P, I, D, P, P, P],
    "chg_joint_dos": [P, I, I, I, I, P, P, I, P, I, P, I, D, P, P, P],
    "chg_structure_factors": [P, P, P, P, P, P, P, P, I, I, I, D, P, P],
    "chg_broadened_spectrum": [P, P, I, I, I, I64, I, I64, P, I, D, P, I64, P, P],
    "chg_phonon_interaction": [P, P, P, P, P, P, I, I, I, I, I, P, P, I, P, I, D, P, I64, P, P],
    "chg_imag_self_energy": [P, I, I, I, I, P, I, P, P, I, P, P, I, D, P, I64, P, P],
    "chg_collision_rows": [P, I, I, I, I, P, I, P, P, I, P, P, I, D, P, I64, P, P],
    "chg_self_energy_spectrum": [P, I, I, I, I, P, I, P, I, P, I, P, P, I, D, P, I64, P, P],
    "chg_coherence_conductivity": [P, P, P, P, P, P, I, I, I, D, P, I64, P, P],
    "chg_isotope_scattering": [P, P, I, I, I, I, P, P, I, P, I, P, D, P, P, I64, P],
    "chg_sample_displacements": [P, P, I, P, P, P, P, I64, I64, I64, I, P, I64, P, P, P],
    "chg_displacement_moments": [P, P, P, P, I, I, I, P, I64, P, P],
}

# CHG_{DOS,TD,JDOS}_MAX_CHUNKS of include/chgnet_b200.h: the scratch blocks chg_tetrahedron_dos,
# chg_thermal_displacements and chg_joint_dos may fill (tests/test_abi_symbols.py ties the copies to the header)
DOS_MAX_CHUNKS = 512
TD_MAX_CHUNKS = 128
JDOS_MAX_CHUNKS = 64
# CHG_SQW_MAX_CHUNKS: the most chunks chg_broadened_spectrum uses (tests/test_structure_factor_spec.py ties it to the
# header); the call also uses no more chunks than its work argument holds
SQW_MAX_CHUNKS = 64


def sqw_scratch_doubles(n_rows, n_modes, n_t, row0, group_size, n_freq):
    """The scratch ``CudaKernels.broadened_spectrum`` allocates for one call: n_t x (groups the rows [row0, row0 +
    n_rows) touch) x n_freq doubles per chunk, for at most one chunk per 32 items of the largest group (the kernel's
    smallest tile) and at most ``SQW_MAX_CHUNKS``."""
    if n_rows <= 0:
        return 0
    groups = (row0 + n_rows - 1) // group_size - row0 // group_size + 1
    chunks = max(1, min(SQW_MAX_CHUNKS, -(-min(group_size, n_rows) * n_modes // 32)))
    return chunks * n_t * groups * n_freq


# CHG_ISE_MAX_CHUNKS: the most chunks chg_imag_self_energy's partial sums use (tests/test_three_phonon_spec.py ties it
# to the header)
ISE_MAX_CHUNKS = 64


def ph3_scratch_doubles(n_q1, n_prim, n_super):
    """The scratch of one ``chg_phonon_interaction`` call: the image averages of q1 and q2, 2 n_q1 n_prim n_super
    complex, and two [n_q1, 3n, 3n, 3n] complex buffers."""
    return 4 * n_q1 * (n_prim * n_super + (3 * n_prim) ** 3)


def ise_scratch_doubles(n_q1, n_band, n_t):
    """The scratch of one ``chg_imag_self_energy`` call: the tetrahedron weights [n_q1, n_band^3, 2] and
    ``ISE_MAX_CHUNKS`` chunks of [n_t, n_band] partial sums."""
    return 2 * n_q1 * n_band**3 + ISE_MAX_CHUNKS * n_t * n_band


def collision_scratch_doubles(n_q1, n_band):
    """The scratch of one ``chg_collision_rows`` call: the tetrahedron weights g2, g1+ and g1-, three [n_q1, n_band^3]
    planes."""
    return 3 * n_q1 * n_band**3


# CHG_SE_MAX_CHUNKS: the most chunks chg_self_energy_spectrum's partial sums use (tests/test_spectral_function_spec.py
# ties it to the header)
SE_MAX_CHUNKS = 128


def se_scratch_doubles(n_band, n_freq, n_t):
    """The scratch of one ``chg_self_energy_spectrum`` call: ``SE_MAX_CHUNKS`` chunks of [n_t, n_band, n_freq] partial
    sums (no per-q1 part)."""
    return SE_MAX_CHUNKS * n_t * n_band * n_freq


# CHG_WIGNER_MAX_CHUNKS: the most chunks chg_coherence_conductivity's partial sums use (tests/test_wigner_spec.py ties
# it to the header)
WIGNER_MAX_CHUNKS = 256


def coherence_scratch_doubles(n_q, n_band, n_t):
    """The scratch of one ``chg_coherence_conductivity`` call: W = dD/dQ E and the velocity operator V, two
    [n_q, 3, n_band, n_band] complex buffers, and ``WIGNER_MAX_CHUNKS`` chunks of [n_t, 6] partial sums."""
    return 12 * n_q * n_band**2 + WIGNER_MAX_CHUNKS * n_t * 6


# CHG_ISO_MAX_CHUNKS: the most chunks chg_isotope_scattering's partial sums use (tests/test_isotope_spec.py ties it to
# the header)
ISO_MAX_CHUNKS = 128


def isotope_scratch_doubles(n_target, n_q, n_band):
    """The scratch of one ``chg_isotope_scattering`` call: the overlaps [n_target, n_q, n_band, n_band] and
    ``ISO_MAX_CHUNKS`` chunks of [n_target, n_band] partial sums."""
    return n_target * n_q * n_band**2 + ISO_MAX_CHUNKS * n_target * n_band


def sampler_scratch_doubles(n_samples, n_modes):
    """The scratch of one ``chg_sample_displacements`` call: the amplitude-scaled normal variates [n_samples,
    n_modes]."""
    return n_samples * n_modes


def moments_scratch_doubles(n_samples, n_prim, n_atoms):
    """The scratch of one ``chg_displacement_moments`` call: the running sums and one slot per sample of the
    18 n_prim n_atoms + 2 folded moments."""
    return (1 + n_samples) * (18 * n_prim * n_atoms + 2)

_lib = None


class ChgnetB200Error(RuntimeError):
    pass


def _mesh_args(name, mesh, freqs, tetrahedra, f64_names, f64_tensors):
    """(n1, n2, n3) of ``mesh``, checking f64_tensors (None skipped), tetrahedra [6, 4, 3] int32 and freqs."""
    n1, n2, n3 = (int(n) for n in mesh)
    if any(t is not None and t.dtype != torch.float64 for t in f64_tensors):
        raise ChgnetB200Error(f"{name}: {f64_names} must be float64")
    if tetrahedra.dtype != torch.int32 or tuple(tetrahedra.shape) != (6, 4, 3):
        raise ChgnetB200Error(f"{name}: tetrahedra must be int32 [6, 4, 3]")
    if freqs.shape[0] != n1 * n2 * n3:
        raise ChgnetB200Error(f"{name}: freqs must be [{n1 * n2 * n3}, n_band]")
    return n1, n2, n3


def _chunk_scratch(max_chunks, per_chunk, device):
    """fp64 scratch for at most ``max_chunks`` chunks of ``per_chunk`` partial sums."""
    return torch.empty(max_chunks * max(per_chunk, 1), dtype=torch.float64, device=device)


def load_library(path: str | None = None) -> ctypes.CDLL:
    """dlopen the kernel library; raises if it has not been built."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise ChgnetB200Error(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C chgnet_b200/csrc`). chgnet_b200 has no CPU or PyTorch fallback."
        )
    lib = ctypes.CDLL(path)
    lib.chg_last_error.restype = c_char_p
    lib.chg_last_error.argtypes = []
    lib.chg_abi_version.restype = c_int32
    lib.chg_abi_version.argtypes = []
    lib.chg_launch_count.restype = c_int64
    lib.chg_launch_count.argtypes = []
    lib.chg_set_option.restype = c_int32
    lib.chg_set_option.argtypes = [c_char_p, c_int32]
    lib.chg_wgrad_workspace_floats.restype = c_int64
    lib.chg_wgrad_workspace_floats.argtypes = [c_int32]
    lib.chg_gated_fused_workspace_floats.restype = c_int64
    lib.chg_gated_fused_workspace_floats.argtypes = [c_int32]
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype = c_int32
        fn.argtypes = argtypes
    _lib = lib
    return lib


def _p(t: Tensor | None):
    if t is None:
        return None
    return t.data_ptr()


class CudaKernels:
    """Python face of the C ABI: one method per entry point, tensors in, nothing returned."""

    name = "cuda"

    def __init__(self, device: torch.device | str | int | None = None) -> None:
        """``device``: the CUDA device whose tensors this object will be handed (default: the current one).
        Every launch runs with that device current and on ITS current stream, whatever the process's
        current device is (``CHGNet.load(use_device='cuda:1')`` in a process sitting on cuda:0)."""
        self.lib = load_library()
        if not torch.cuda.is_available():
            raise ChgnetB200Error("chgnet_b200 needs a CUDA device (H100 / sm_90a); none is visible")
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise ChgnetB200Error(f"chgnet_b200 kernels run on CUDA devices only (got {dev})")
        self.device_index = torch.cuda.current_device() if dev.index is None else dev.index

    # ------------------------------------------------------------------
    def _stream(self):
        return torch.cuda.current_stream(self.device_index).cuda_stream

    def _call(self, name: str, *args) -> None:
        if torch.cuda.current_device() != self.device_index:
            with torch.cuda.device(self.device_index):
                return self._call(name, *args)
        rc = getattr(self.lib, name)(*args, self._stream())
        if rc != 0:
            raise ChgnetB200Error(f"{name} failed ({rc}): {self.lib.chg_last_error().decode()}")

    @staticmethod
    def _chk(*tensors: Tensor | None) -> None:
        for t in tensors:
            if t is not None and (not t.is_cuda or not t.is_contiguous()):
                raise ChgnetB200Error("kernel arguments must be contiguous CUDA tensors")

    def set_option(self, name: str, value: int) -> None:
        """A/B switches (include/chgnet_b200.h): 'linear_impl' 0 FFMA | 1 wgmma | 2 wgmma (as 1) |
        3 warp-specialised wgmma + TMA tensor maps (default),
        'gated_impl' 3 fused warp-specialised wgmma message + aggregation (default) | 0 FFMA 4x8 | 1 wgmma | 2 FFMA 8x8."""
        if self.lib.chg_set_option(name.encode(), int(value)) != 0:
            raise ChgnetB200Error(self.lib.chg_last_error().decode())

    @property
    def launches(self) -> int:
        return int(self.lib.chg_launch_count())

    # ------------------------------------------------------------------ kernels
    def embed_atoms(self, z, emb, x):
        self._chk(z, emb, x)
        self._call("chg_embed_atoms", _p(z), _p(emb), z.shape[0], _p(x))

    def edge_geometry(self, frac, lattice, owner, center, nbr, image, rvec, dist, rhat):
        self._chk(frac, lattice, owner, center, nbr, image, rvec, dist, rhat)
        self._call("chg_edge_geometry", _p(frac), _p(lattice), _p(owner), _p(center), _p(nbr), _p(image),
                   center.shape[0], _p(rvec), _p(dist), _p(rhat))

    def bond_basis_embed(self, dist, u2d, freq_ag, freq_bg, rc_ag, rc_bg, p, w3t, e0, wag, wbg, basis_out=None):
        self._chk(dist, u2d, freq_ag, freq_bg, w3t, e0, wag, wbg, basis_out)
        self._call("chg_bond_basis_embed", _p(dist), _p(u2d), u2d.shape[0], _p(freq_ag), _p(freq_bg),
                   freq_ag.shape[0], float(rc_ag), float(rc_bg), int(p), _p(w3t), _p(e0), _p(wag), _p(wbg),
                   _p(basis_out))

    def bond_basis_bwd(self, dist, u2d, freq_ag, freq_bg, rc_ag, rc_bg, p, w3, g_e0, g_wag, g_wbg, g_dist,
                       g_freq=None):
        self._chk(dist, u2d, freq_ag, freq_bg, w3, g_e0, g_wag, g_wbg, g_dist, g_freq)
        self._call("chg_bond_basis_bwd", _p(dist), _p(u2d), u2d.shape[0], _p(freq_ag), _p(freq_bg),
                   freq_ag.shape[0], float(rc_ag), float(rc_bg), int(p), _p(w3), _p(g_e0), _p(g_wag), _p(g_wbg),
                   _p(g_dist), _p(g_freq))

    def angle_basis_embed(self, rhat, ang_di, ang_dj, freq, wt, a0, basis_out=None):
        self._chk(rhat, ang_di, ang_dj, freq, wt, a0, basis_out)
        self._call("chg_angle_basis_embed", _p(rhat), _p(ang_di), _p(ang_dj), ang_di.shape[0], _p(freq),
                   freq.shape[0], _p(wt), _p(a0), _p(basis_out))

    def angle_basis_bwd(self, rhat, ang_di, ang_dj, freq, w, g_a0, g_rhat, g_freq=None):
        self._chk(rhat, ang_di, ang_dj, freq, w, g_a0, g_rhat, g_freq)
        self._call("chg_angle_basis_bwd", _p(rhat), _p(ang_di), _p(ang_dj), ang_di.shape[0], _p(freq),
                   freq.shape[0], _p(w), _p(g_a0), _p(g_rhat), _p(g_freq))

    def linear(self, x, wt, bias, residual, y, x_rows=None, y_rows=None):
        self._chk(x, wt, bias, residual, y, x_rows, y_rows)
        m = x_rows.shape[0] if x_rows is not None else x.shape[0]
        self._call("chg_linear", _p(x), _p(x_rows), m, x.shape[1], _p(wt), _p(bias), _p(residual), _p(y_rows),
                   wt.shape[1], _p(y))

    def gather_rows(self, src, idx, dst):
        self._chk(src, idx, dst)
        self._call("chg_gather_rows", _p(src), _p(idx), idx.shape[0], src.shape[1], _p(dst))

    def scatter_rows(self, src, idx, dst):
        self._chk(src, idx, dst)
        self._call("chg_scatter_rows", _p(src), _p(idx), idx.shape[0], src.shape[1], _p(dst))

    def atom_conv_fwd(self, pcn, pe, wag, center, nbr, d2u, w2t, b2, ln, msg, save_p, save_pre=None):
        self._chk(pcn, pe, wag, center, nbr, d2u, w2t, b2, ln, msg, save_p, save_pre)
        self._call("chg_atom_conv_fwd", _p(pcn), _p(pe), _p(wag), _p(center), _p(nbr), _p(d2u), center.shape[0],
                   _p(w2t), _p(b2), _p(ln), _p(msg), _p(save_p), _p(save_pre))

    def atom_conv_bwd(self, pcn, pe, wag, center, nbr, d2u, save_p, g_agg, w2, ln, g_pre, g_w, g_p=None, g_ln=None):
        self._chk(pcn, pe, wag, center, nbr, d2u, save_p, g_agg, w2, ln, g_pre, g_w, g_p, g_ln)
        self._call("chg_atom_conv_bwd", _p(pcn), _p(pe), _p(wag), _p(center), _p(nbr), _p(d2u), center.shape[0],
                   _p(save_p), _p(g_agg), _p(w2), _p(ln), _p(g_pre), _p(g_w), _p(g_p), _p(g_ln))

    def _fused_work(self, n_rows: int, device) -> Tensor:
        """Grow-only scratch of the fused message + aggregation kernels (strip partials; the message itself
        for the unfused A/B implementations)."""
        need = int(self.lib.chg_gated_fused_workspace_floats(int(n_rows)))
        ws = getattr(self, "_fws", None)
        if ws is None or ws.device != device or ws.numel() < need:
            ws = torch.empty(need, dtype=torch.float32, device=device)
            self._fws = ws
        return ws

    def atom_conv_fused(self, pcn, pe, wag, center, nbr, d2u, ptr_c, w2t, b2, ln, agg, save_p):
        self._chk(pcn, pe, wag, center, nbr, d2u, ptr_c, w2t, b2, ln, agg, save_p)
        self._call("chg_atom_conv_fused", _p(pcn), _p(pe), _p(wag), _p(center), _p(nbr), _p(d2u), _p(ptr_c), center.shape[0],
                   agg.shape[0], _p(w2t), _p(b2), _p(ln), _p(agg), _p(save_p), _p(self._fused_work(center.shape[0], agg.device)))

    def bond_conv_fused(self, pij, px, pa, wbg, ang_atom, ang_i, ang_j, ptr_i, w2t, b2, ln, agg, save_pre, save_p):
        self._chk(pij, px, pa, wbg, ang_atom, ang_i, ang_j, ptr_i, w2t, b2, ln, agg, save_pre, save_p)
        self._call("chg_bond_conv_fused", _p(pij), _p(px), _p(pa), _p(wbg), _p(ang_atom), _p(ang_i), _p(ang_j), _p(ptr_i),
                   ang_i.shape[0], agg.shape[0], _p(w2t), _p(b2), _p(ln), _p(agg), _p(save_pre), _p(save_p),
                   _p(self._fused_work(ang_i.shape[0], agg.device)))

    def segment_sum(self, data, perm, ptr, accumulate, out):
        self._chk(data, perm, ptr)
        if not out.is_cuda or out.stride(1) != 1:
            raise ChgnetB200Error("segment_sum output must be a CUDA tensor with unit column stride")
        n_items = data.shape[0] if perm is None else perm.shape[0]
        self._call("chg_segment_sum", _p(data), data.shape[1], _p(perm), _p(ptr), ptr.shape[0] - 1, n_items,
                   int(accumulate), _p(out), out.stride(0))

    def bond_conv_fwd(self, pij, px, pa, wbg, ang_atom, ang_i, ang_j, w2t, b2, ln, upd, save_pre, save_p):
        self._chk(pij, px, pa, wbg, ang_atom, ang_i, ang_j, w2t, b2, ln, upd, save_pre, save_p)
        self._call("chg_bond_conv_fwd", _p(pij), _p(px), _p(pa), _p(wbg), _p(ang_atom), _p(ang_i), _p(ang_j),
                   ang_i.shape[0], _p(w2t), _p(b2), _p(ln), _p(upd), _p(save_pre), _p(save_p))

    def bond_conv_bwd(self, save_pre, save_p, wbg, ang_i, ang_j, g_agg, w2, ln, g_pre, gw_i, gw_j, g_p=None,
                      g_ln=None):
        self._chk(save_pre, save_p, wbg, ang_i, ang_j, g_agg, w2, ln, g_pre, gw_i, gw_j, g_p, g_ln)
        self._call("chg_bond_conv_bwd", _p(save_pre), _p(save_p), _p(wbg), _p(ang_i), _p(ang_j), ang_i.shape[0],
                   _p(g_agg), _p(w2), _p(ln), _p(g_pre), _p(gw_i), _p(gw_j), _p(g_p), _p(g_ln))

    def angle_update_fwd(self, pij, px, pa, ang, ang_atom, ang_i, ang_j, ln, ang_new, save_p):
        self._chk(pij, px, pa, ang, ang_atom, ang_i, ang_j, ln, ang_new, save_p)
        self._call("chg_angle_update_fwd", _p(pij), _p(px), _p(pa), _p(ang), _p(ang_atom), _p(ang_i), _p(ang_j),
                   ang_i.shape[0], _p(ln), _p(ang_new), _p(save_p))

    def angle_update_bwd(self, save_p, g_ang_in, ln, g_pre, g_ln=None):
        self._chk(save_p, g_ang_in, ln, g_pre, g_ln)
        self._call("chg_angle_update_bwd", _p(save_p), _p(g_ang_in), save_p.shape[0], _p(ln), _p(g_pre), _p(g_ln))

    # ------------------------------------------------------------------ training
    @staticmethod
    def _chk_rows(*tensors: Tensor | None) -> None:
        for t in tensors:
            if t is not None and (not t.is_cuda or t.stride(-1) != 1):
                raise ChgnetB200Error("kernel arguments must be CUDA tensors with unit column stride")

    def _workspace(self, n_out: int, device) -> Tensor:
        ws = getattr(self, "_ws", None)
        if ws is None or ws.device != device:
            need = max(int(self.lib.chg_wgrad_workspace_floats(n)) for n in (64, 128, 256))
            ws = torch.empty(need, dtype=torch.float32, device=device)
            self._ws = ws
        return ws

    def wgrad(self, x, g, out, colsum=None, x_rows=None, g_rows=None, x_silu=False, x2=None):
        self._chk_rows(x, g, out, x2)
        self._chk(colsum, x_rows, g_rows)
        if x2 is not None and x2.stride(0) != x.stride(0):
            raise ChgnetB200Error("wgrad: x2 must have the row stride of x")
        m = x_rows.shape[0] if x_rows is not None else (g_rows.shape[0] if g_rows is not None else x.shape[0])
        self._call("chg_wgrad", _p(x), _p(x2), x.stride(0), _p(x_rows), int(bool(x_silu)), _p(g), g.stride(0), _p(g_rows), m,
                   out.shape[1], _p(out), out.stride(0), _p(colsum), _p(self._workspace(out.shape[1], x.device)))

    def colsum(self, a, out, b=None, rowscale=None):
        self._chk_rows(a, b)
        self._chk(out, rowscale)
        self._call("chg_colsum", _p(a), a.stride(0), _p(b), b.stride(0) if b is not None else 0, _p(rowscale),
                   a.shape[0], a.shape[1], _p(out))

    def readout_bwd(self, x, ln, mlp_wt, mlp_w, mlp_b, w_last, seed, g_x, h_all, gz_all, g_h0, xhat):
        self._chk(x, ln, mlp_wt, mlp_w, mlp_b, w_last, seed, g_x, h_all, gz_all, g_h0, xhat)
        self._call("chg_readout_bwd", _p(x), x.shape[0], _p(ln), _p(mlp_wt), _p(mlp_w), _p(mlp_b), mlp_wt.shape[0],
                   _p(w_last), _p(seed), _p(g_x), _p(h_all), _p(gz_all), _p(g_h0), _p(xhat))

    def magmom_bwd(self, x, w, b, g_m, g_x, g_lin):
        self._chk(x, w, g_m, g_x, g_lin)
        self._call("chg_magmom_bwd", _p(x), x.shape[0], _p(w), float(b), _p(g_m), _p(g_x), _p(g_lin))

    def loss_terms(self, pred, target, kind, delta, g_pred, sums):
        self._chk(pred, target, g_pred, sums)
        self._call("chg_loss_terms", _p(pred), _p(target), pred.numel(), int(kind), float(delta), _p(g_pred), _p(sums))

    # ------------------------------------------------------------------ second order
    def edge_tangent(self, rvec, dist, rhat, center, nbr, owner, u_atom, w_graph, ddist, drhat):
        self._chk(rvec, dist, rhat, center, nbr, owner, u_atom, w_graph, ddist, drhat)
        self._call("chg_edge_tangent", _p(rvec), _p(dist), _p(rhat), _p(center), _p(nbr), _p(owner), _p(u_atom),
                   _p(w_graph), center.shape[0], _p(ddist), _p(drhat))

    def bond_basis_tangent(self, dist, ddist, u2d, freq_ag, freq_bg, rc_ag, rc_bg, p, w3t, e0d, wagd, wbgd, tbasis):
        self._chk(dist, ddist, u2d, freq_ag, freq_bg, w3t, e0d, wagd, wbgd, tbasis)
        self._call("chg_bond_basis_tangent", _p(dist), _p(ddist), _p(u2d), u2d.shape[0], _p(freq_ag), _p(freq_bg),
                   freq_ag.shape[0], float(rc_ag), float(rc_bg), int(p), _p(w3t), _p(e0d), _p(wagd), _p(wbgd), _p(tbasis))

    def bond_basis_bwd2(self, dist, ddist, u2d, freq_ag, freq_bg, rc_ag, rc_bg, p, w3, lam_e0, lam_wag, lam_wbg, g_freq):
        self._chk(dist, ddist, u2d, freq_ag, freq_bg, w3, lam_e0, lam_wag, lam_wbg, g_freq)
        self._call("chg_bond_basis_bwd2", _p(dist), _p(ddist), _p(u2d), u2d.shape[0], _p(freq_ag), _p(freq_bg),
                   freq_ag.shape[0], float(rc_ag), float(rc_bg), int(p), _p(w3), _p(lam_e0), _p(lam_wag), _p(lam_wbg),
                   _p(g_freq))

    def angle_basis_tangent(self, rhat, drhat, ang_di, ang_dj, freq, wt, a0d, tbasis):
        self._chk(rhat, drhat, ang_di, ang_dj, freq, wt, a0d, tbasis)
        self._call("chg_angle_basis_tangent", _p(rhat), _p(drhat), _p(ang_di), _p(ang_dj), ang_di.shape[0], _p(freq),
                   freq.shape[0], _p(wt), _p(a0d), _p(tbasis))

    def angle_basis_bwd2(self, rhat, drhat, ang_di, ang_dj, freq, w, lam_a0, g_freq):
        self._chk(rhat, drhat, ang_di, ang_dj, freq, w, lam_a0, g_freq)
        self._call("chg_angle_basis_bwd2", _p(rhat), _p(drhat), _p(ang_di), _p(ang_dj), ang_di.shape[0], _p(freq),
                   freq.shape[0], _p(w), _p(lam_a0), _p(g_freq))

    def bond_basis_hvp(self, dist, ddist, u2d, freq_ag, freq_bg, rc_ag, rc_bg, p, w3, lam_e0, lam_wag, lam_wbg, g_dist):
        self._chk(dist, ddist, u2d, freq_ag, freq_bg, w3, lam_e0, lam_wag, lam_wbg, g_dist)
        self._call("chg_bond_basis_hvp", _p(dist), _p(ddist), _p(u2d), u2d.shape[0], _p(freq_ag), _p(freq_bg),
                   freq_ag.shape[0], float(rc_ag), float(rc_bg), int(p), _p(w3), _p(lam_e0), _p(lam_wag), _p(lam_wbg),
                   _p(g_dist))

    def angle_basis_hvp(self, rhat, drhat, ang_di, ang_dj, freq, w, lam_a0, g_rhat):
        self._chk(rhat, drhat, ang_di, ang_dj, freq, w, lam_a0, g_rhat)
        self._call("chg_angle_basis_hvp", _p(rhat), _p(drhat), _p(ang_di), _p(ang_dj), ang_di.shape[0], _p(freq),
                   freq.shape[0], _p(w), _p(lam_a0), _p(g_rhat))

    def edge_tangent_bwd(self, dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, force):
        self._chk(dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, force)
        self._call("chg_edge_tangent_bwd", _p(dist), _p(rhat), _p(ddist), _p(drhat), _p(lam_dist), _p(lam_rhat), _p(d2u),
                   _p(u2d), _p(center), _p(nbr), center.shape[0], _p(force))

    def edge_tangent_bwd_virial(self, rvec, dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, owner,
                                force, virial):
        self._chk(rvec, dist, rhat, ddist, drhat, lam_dist, lam_rhat, d2u, u2d, center, nbr, owner, force, virial)
        self._call("chg_edge_tangent_bwd_virial", _p(rvec), _p(dist), _p(rhat), _p(ddist), _p(drhat), _p(lam_dist),
                   _p(lam_rhat), _p(d2u), _p(u2d), _p(center), _p(nbr), _p(owner), center.shape[0], _p(force), _p(virial))

    def dynamical_matrices(self, fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, dyn):
        """dyn [Q, 3n, 3n] complex128 (overwritten) = D(q) of the compact force constants fc [n, N, 3, 3] (fp64)."""
        self._chk(fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, dyn)
        if dyn.dtype != torch.complex128 or fc.dtype != torch.float64 or qpoints.dtype != torch.float64:
            raise ChgnetB200Error("dynamical_matrices: fc and qpoints must be float64, dyn complex128")
        self._call("chg_dynamical_matrices", _p(fc), _p(img_ptr), _p(img_vec), _p(s2p), _p(inv_sqrt_m), fc.shape[0],
                   fc.shape[1], _p(qpoints), qpoints.shape[0], _p(dyn))

    def dynamical_matrix_derivatives(self, fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, prim_lattice, ddyn):
        """ddyn [Q, 3, 3n, 3n] complex128 (overwritten) = dD/dQ_c, Q = q inv(prim_lattice)^T (1/A, no 2 pi), for the
        arguments of ``dynamical_matrices`` and the primitive lattice [3, 3] (fp64, rows are lattice vectors, A)."""
        self._chk(fc, img_ptr, img_vec, s2p, inv_sqrt_m, qpoints, prim_lattice, ddyn)
        if (ddyn.dtype != torch.complex128 or fc.dtype != torch.float64 or qpoints.dtype != torch.float64
                or prim_lattice.dtype != torch.float64):
            raise ChgnetB200Error("dynamical_matrix_derivatives: fc, qpoints and prim_lattice must be float64, "
                                  "ddyn complex128")
        n3 = 3 * fc.shape[0]
        if tuple(prim_lattice.shape) != (3, 3) or tuple(ddyn.shape) != (qpoints.shape[0], 3, n3, n3):
            raise ChgnetB200Error(f"dynamical_matrix_derivatives: prim_lattice must be [3, 3] and ddyn "
                                  f"[{qpoints.shape[0]}, 3, {n3}, {n3}]")
        self._call("chg_dynamical_matrix_derivatives", _p(fc), _p(img_ptr), _p(img_vec), _p(s2p), _p(inv_sqrt_m),
                   fc.shape[0], fc.shape[1], _p(qpoints), qpoints.shape[0], _p(prim_lattice), _p(ddyn))

    def tetrahedron_dos(self, freqs, mesh, tetrahedra, omega, dos, idos, proj=None, pdos=None):
        """Linear tetrahedron DOS on the full Gamma-centred ``mesh`` (n1, n2, n3): freqs [n1 n2 n3, n_band] fp64
        (ascending per q), tetrahedra [6, 4, 3] int32 corner offsets, omega [F] fp64; writes dos [F], idos [F] and,
        with proj [n1 n2 n3, n_band, S], pdos [S, F] (all fp64)."""
        self._chk(freqs, tetrahedra, omega, dos, idos, proj, pdos)
        n1, n2, n3 = _mesh_args("tetrahedron_dos", mesh, freqs, tetrahedra, "freqs, omega, proj and the outputs",
                                (freqs, omega, dos, idos, proj, pdos))
        n_q, n_band = freqs.shape
        n_f = omega.shape[0]
        if tuple(dos.shape) != (n_f,) or tuple(idos.shape) != (n_f,):
            raise ChgnetB200Error(f"tetrahedron_dos: dos and idos must be [{n_f}]")
        n_proj = 0
        if proj is not None:
            n_proj = proj.shape[2]
            if tuple(proj.shape[:2]) != (n_q, n_band) or pdos is None or tuple(pdos.shape) != (n_proj, n_f):
                raise ChgnetB200Error(f"tetrahedron_dos: proj must be [{n_q}, {n_band}, S] and pdos [S, {n_f}]")
        work = _chunk_scratch(DOS_MAX_CHUNKS, (2 + n_proj) * n_f, freqs.device)
        self._call("chg_tetrahedron_dos", _p(freqs), n_band, n1, n2, n3, _p(tetrahedra), _p(proj), n_proj, _p(omega),
                   n_f, _p(dos), _p(idos), _p(pdos if proj is not None else None), _p(work))

    def thermal_displacements(self, freqs, eigvecs, temperatures, cutoff_thz, acc):
        """acc [T, n_prim, 6] fp64 += sum over (q, mode) of w(nu, T) Re(e e^H) per atom in Voigt order (xx, yy, zz,
        yz, xz, xy), w = (1 + 2 / expm1(h nu / k T)) / nu for nu >= cutoff_thz and 0 otherwise: freqs [Q, 3n] THz
        (fp64, signed), eigvecs [Q, mode, 3n] complex128 (mode-major: ``e.mT`` of eigh's eigenvectors), temperatures
        [T] K (fp64)."""
        self._chk(freqs, eigvecs, temperatures, acc)
        f64 = torch.float64
        if (freqs.dtype != f64 or temperatures.dtype != f64 or acc.dtype != f64
                or eigvecs.dtype != torch.complex128):
            raise ChgnetB200Error("thermal_displacements: freqs, temperatures and acc must be float64, eigvecs "
                                  "complex128")
        n_q, n3 = freqs.shape
        n_t = temperatures.shape[0]
        if (n3 % 3 or tuple(eigvecs.shape) != (n_q, n3, n3) or temperatures.dim() != 1
                or tuple(acc.shape) != (n_t, n3 // 3, 6)):
            raise ChgnetB200Error(f"thermal_displacements: freqs must be [Q, 3n], eigvecs [{n_q}, {n3}, {n3}], "
                                  f"temperatures [T] and acc [T, {n3 // 3}, 6]")
        work = _chunk_scratch(TD_MAX_CHUNKS, n_t * (n3 // 3) * 6, freqs.device)
        self._call("chg_thermal_displacements", _p(freqs), _p(eigvecs), n_q, n3 // 3, _p(temperatures), n_t,
                   float(cutoff_thz), _p(work), _p(acc))

    def joint_dos(self, freqs, mesh, tetrahedra, targets, omega, temperatures, cutoff_thz, out):
        """Two-phonon joint densities of states on the full Gamma-centred ``mesh`` (n1, n2, n3): freqs [n1 n2 n3,
        n_band] fp64 THz (ascending per q), tetrahedra [6, 4, 3] int32, targets [Q] int32 mesh indices, omega [Q, F]
        fp64 THz (the frequency points of each target), temperatures [T] fp64 K or None; writes out [Q, 1 + T, 2, F]
        fp64 (slot 0: D2 classes 1 and 2; slot 1 + t: N2 at temperatures[t]), modes below cutoff_thz left out."""
        self._chk(freqs, tetrahedra, targets, omega, temperatures, out)
        n1, n2, n3 = _mesh_args("joint_dos", mesh, freqs, tetrahedra, "freqs, omega, temperatures and out",
                                (freqs, omega, temperatures, out))
        if targets.dtype != torch.int32 or targets.dim() != 1:
            raise ChgnetB200Error("joint_dos: targets must be int32 [Q]")
        n_band = freqs.shape[1]
        n_target = targets.shape[0]
        n_t = 0 if temperatures is None else temperatures.shape[0]
        if temperatures is not None and temperatures.dim() != 1:
            raise ChgnetB200Error("joint_dos: temperatures must be [T]")
        if omega.dim() != 2 or omega.shape[0] != n_target:
            raise ChgnetB200Error(f"joint_dos: omega must be [{n_target}, F]")
        n_f = omega.shape[1]
        if tuple(out.shape) != (n_target, 1 + n_t, 2, n_f):
            raise ChgnetB200Error(f"joint_dos: out must be [{n_target}, {1 + n_t}, 2, {n_f}]")
        work = _chunk_scratch(JDOS_MAX_CHUNKS, n_target * (1 + n_t) * 2 * n_f, freqs.device)
        self._call("chg_joint_dos", _p(freqs), n_band, n1, n2, n3, _p(tetrahedra), _p(targets), n_target, _p(omega),
                   n_f, _p(temperatures), n_t, float(cutoff_thz), _p(out), _p(work))

    def structure_factors(self, freqs, eigvecs, kcart, gvec, frac, coef, u, temperatures, cutoff_thz, out):
        """out [T, Q, 3n, 2] fp64 (overwritten) = (S+, S-) of every row and mode, coherent one-phonon structure
        factors in A^2 x coef^2 (``chg_structure_factors``): freqs [Q, 3n] THz (signed), eigvecs [Q, mode, 3n]
        complex128 (mode-major: ``e.mT`` of eigh's eigenvectors), kcart [Q, 3] Cartesian K (1/A, 2 pi included), gvec
        [Q, 3] reduced G, frac [n, 3] fractional positions, coef [n] = b / sqrt(m), u [T, n, 6] Voigt U (A^2) or None
        for no Debye-Waller factor, temperatures [T] K (all fp64); modes below cutoff_thz get 0."""
        self._chk(freqs, eigvecs, kcart, gvec, frac, coef, u, temperatures, out)
        f64 = torch.float64
        if (any(t is not None and t.dtype != f64 for t in (freqs, kcart, gvec, frac, coef, u, temperatures, out))
                or eigvecs.dtype != torch.complex128):
            raise ChgnetB200Error("structure_factors: eigvecs must be complex128 and every other tensor float64")
        n_q, n3 = freqs.shape
        n_prim, n_t = n3 // 3, temperatures.shape[0]
        if (n3 % 3 or tuple(eigvecs.shape) != (n_q, n3, n3) or tuple(kcart.shape) != (n_q, 3)
                or tuple(gvec.shape) != (n_q, 3) or tuple(frac.shape) != (n_prim, 3) or tuple(coef.shape) != (n_prim,)
                or temperatures.dim() != 1 or (u is not None and tuple(u.shape) != (n_t, n_prim, 6))
                or tuple(out.shape) != (n_t, n_q, n3, 2)):
            raise ChgnetB200Error(f"structure_factors: freqs must be [Q, 3n], eigvecs [{n_q}, {n3}, {n3}], kcart and "
                                  f"gvec [{n_q}, 3], frac [{n_prim}, 3], coef [{n_prim}], temperatures [T], u None or "
                                  f"[T, {n_prim}, 6] and out [T, {n_q}, {n3}, 2]")
        self._call("chg_structure_factors", _p(freqs), _p(eigvecs), _p(kcart), _p(gvec), _p(frac), _p(coef), _p(u),
                   _p(temperatures), n_t, n_q, n_prim, float(cutoff_thz), _p(out))

    def broadened_spectrum(self, freqs, weights, row0, group_size, omega, sigma, out):
        """out [T, n_groups, F] fp64 += (1 / group_size) sum over the rows of each group and their modes of
        S+ g(omega - nu) + S- g(omega + nu), g the normalised Gaussian of standard deviation sigma (THz) cut at
        8 sigma (``chg_broadened_spectrum``): freqs [Q, 3n] THz are the rows [row0, row0 + Q) of the map, row r in group
        r // group_size; weights [T, Q, 3n, 2] (S+, S-) as ``structure_factors`` writes them; omega [F] THz."""
        self._chk(freqs, weights, omega, out)
        if any(t.dtype != torch.float64 for t in (freqs, weights, omega, out)):
            raise ChgnetB200Error("broadened_spectrum: freqs, weights, omega and out must be float64")
        n_q, n3 = freqs.shape
        n_t, n_f = weights.shape[0], omega.shape[0]
        row0, group_size = int(row0), int(group_size)
        if (tuple(weights.shape) != (n_t, n_q, n3, 2) or omega.dim() != 1 or out.dim() != 3
                or tuple(out.shape[::2]) != (n_t, n_f)):
            raise ChgnetB200Error(f"broadened_spectrum: weights must be [T, {n_q}, {n3}, 2], omega [F] and out "
                                  f"[T, n_groups, F]")
        if n_q == 0:
            return
        work = torch.empty(max(1, sqw_scratch_doubles(n_q, n3, n_t, row0, group_size, n_f)), dtype=torch.float64,
                           device=freqs.device)
        self._call("chg_broadened_spectrum", _p(freqs), _p(weights), n_q, n3, n_t, row0, group_size, out.shape[1],
                   _p(omega), n_f, float(sigma), _p(work), work.numel(), _p(out))

    def phonon_interaction(self, fc3, img_ptr, img_vec, s2p, inv_sqrt_m, frac, mesh, freqs, eigvecs, target, q1,
                           cutoff_thz, out):
        """out [n_q1, 3n, 3n, 3n] fp64 (overwritten) = the interaction strengths P (eV^2) of the target q (mesh index)
        with the q1 of the mesh indices ``q1`` [n_q1] int32 and q2 = q - q1 (``chg_phonon_interaction``): fc3 [n, N, N,
        3, 3, 3] eV/A^3, img_ptr, img_vec, s2p and inv_sqrt_m as ``dynamical_matrices`` (the supercell atom-major),
        frac [n, 3] fractional positions, freqs [n1 n2 n3, 3n] THz and eigvecs [n1 n2 n3, mode, 3n] complex128 (mode-
        major) of the full Gamma-centred ``mesh``; modes below cutoff_thz give 0."""
        self._chk(fc3, img_ptr, img_vec, s2p, inv_sqrt_m, frac, freqs, eigvecs, q1, out)
        f64 = torch.float64
        if (any(t.dtype != f64 for t in (fc3, img_vec, inv_sqrt_m, frac, freqs, out))
                or eigvecs.dtype != torch.complex128 or q1.dtype != torch.int32 or s2p.dtype != torch.int32):
            raise ChgnetB200Error("phonon_interaction: eigvecs must be complex128, q1 and s2p int32 and every other "
                                  "tensor float64")
        n1, n2, n3 = (int(n) for n in mesh)
        n_prim, n_super = fc3.shape[0], fc3.shape[1]
        nb, n_q1 = 3 * n_prim, q1.shape[0]
        if (tuple(fc3.shape) != (n_prim, n_super, n_super, 3, 3, 3) or tuple(frac.shape) != (n_prim, 3)
                or tuple(freqs.shape) != (n1 * n2 * n3, nb) or tuple(eigvecs.shape) != (n1 * n2 * n3, nb, nb)
                or q1.dim() != 1 or tuple(out.shape) != (n_q1, nb, nb, nb)):
            raise ChgnetB200Error(f"phonon_interaction: fc3 must be [n, N, N, 3, 3, 3], frac [{n_prim}, 3], freqs "
                                  f"[{n1 * n2 * n3}, {nb}], eigvecs [{n1 * n2 * n3}, {nb}, {nb}], q1 [Q1] and out "
                                  f"[Q1, {nb}, {nb}, {nb}]")
        if n_prim and (n_super % n_prim or not torch.equal(
                s2p, torch.arange(n_super, device=s2p.device, dtype=torch.int32) // (n_super // n_prim))):
            raise ChgnetB200Error("phonon_interaction: the supercell must be atom-major (s2p[j] = j // n_cells)")
        work = torch.empty(max(1, ph3_scratch_doubles(n_q1, n_prim, n_super)), dtype=f64, device=freqs.device)
        self._call("chg_phonon_interaction", _p(fc3), _p(img_ptr), _p(img_vec), _p(s2p), _p(inv_sqrt_m), _p(frac),
                   n_prim, n_super, n1, n2, n3, _p(freqs), _p(eigvecs), int(target), _p(q1), n_q1, float(cutoff_thz),
                   _p(work), work.numel(), _p(out))

    def imag_self_energy(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, gamma):
        """gamma [T, n_band] fp64 += the contribution of the q1 (mesh indices ``q1`` [n_q1] int32) to the imaginary
        self-energy (half width, THz) of the target's modes at w = omega [n_band] (``chg_imag_self_energy``): freqs
        [n1 n2 n3, n_band] THz, tetrahedra [6, 4, 3] int32, p [n_q1, n_band, n_band, n_band] the interaction strengths
        of ``phonon_interaction``, temperatures [T] K; modes below cutoff_thz left out."""
        self._chk(freqs, tetrahedra, omega, q1, p, temperatures, gamma)
        n1, n2, n3 = _mesh_args("imag_self_energy", mesh, freqs, tetrahedra, "freqs, omega, p, temperatures and gamma",
                                (freqs, omega, p, temperatures, gamma))
        nb, n_q1, n_t = freqs.shape[1], q1.shape[0], temperatures.shape[0]
        if (q1.dtype != torch.int32 or q1.dim() != 1 or tuple(omega.shape) != (nb,) or temperatures.dim() != 1
                or tuple(p.shape) != (n_q1, nb, nb, nb) or tuple(gamma.shape) != (n_t, nb)):
            raise ChgnetB200Error(f"imag_self_energy: q1 must be int32 [Q1], omega [{nb}], p [Q1, {nb}, {nb}, {nb}], "
                                  f"temperatures [T] and gamma [T, {nb}]")
        work = torch.empty(max(1, ise_scratch_doubles(n_q1, nb, n_t)), dtype=torch.float64, device=freqs.device)
        self._call("chg_imag_self_energy", _p(freqs), nb, n1, n2, n3, _p(tetrahedra), int(target), _p(omega), _p(q1),
                   n_q1, _p(p), _p(temperatures), n_t, float(cutoff_thz), _p(work), work.numel(), _p(gamma))

    def collision_rows(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, out):
        """out [4, T, n_band, n1 n2 n3, n_band] fp64: the collision-matrix role sums (1/ps) of the target's modes with
        the vertices q1 (mesh indices ``q1`` [n_q1] int32), written at out[:, :, :, q1] and nowhere else
        (``chg_collision_rows``, DESIGN.md section 12.8); the other arguments as ``imag_self_energy``."""
        self._chk(freqs, tetrahedra, omega, q1, p, temperatures, out)
        n1, n2, n3 = _mesh_args("collision_rows", mesh, freqs, tetrahedra, "freqs, omega, p, temperatures and out",
                                (freqs, omega, p, temperatures, out))
        nb, n_q1, n_t = freqs.shape[1], q1.shape[0], temperatures.shape[0]
        if (q1.dtype != torch.int32 or q1.dim() != 1 or tuple(omega.shape) != (nb,) or temperatures.dim() != 1
                or tuple(p.shape) != (n_q1, nb, nb, nb) or tuple(out.shape) != (4, n_t, nb, n1 * n2 * n3, nb)):
            raise ChgnetB200Error(f"collision_rows: q1 must be int32 [Q1], omega [{nb}], p [Q1, {nb}, {nb}, {nb}], "
                                  f"temperatures [T] and out [4, T, {nb}, {n1 * n2 * n3}, {nb}]")
        work = torch.empty(max(1, collision_scratch_doubles(n_q1, nb)), dtype=torch.float64, device=freqs.device)
        self._call("chg_collision_rows", _p(freqs), nb, n1, n2, n3, _p(tetrahedra), int(target), _p(omega), _p(q1),
                   n_q1, _p(p), _p(temperatures), n_t, float(cutoff_thz), _p(work), work.numel(), _p(out))

    def self_energy_spectrum(self, freqs, mesh, tetrahedra, target, omega, q1, p, temperatures, cutoff_thz, gamma):
        """gamma [T, n_band, F] fp64 += the contribution of the q1 (mesh indices ``q1`` [n_q1] int32) to the imaginary
        self-energy (half width, THz) of the target's modes at the points omega [F] (ascending, shared by every band;
        0 below cutoff_thz) (``chg_self_energy_spectrum``); the other arguments as ``imag_self_energy``."""
        self._chk(freqs, tetrahedra, omega, q1, p, temperatures, gamma)
        n1, n2, n3 = _mesh_args("self_energy_spectrum", mesh, freqs, tetrahedra,
                                "freqs, omega, p, temperatures and gamma", (freqs, omega, p, temperatures, gamma))
        nb, n_q1, n_t, n_f = freqs.shape[1], q1.shape[0], temperatures.shape[0], omega.shape[0]
        if (q1.dtype != torch.int32 or q1.dim() != 1 or omega.dim() != 1 or temperatures.dim() != 1
                or tuple(p.shape) != (n_q1, nb, nb, nb) or tuple(gamma.shape) != (n_t, nb, n_f)):
            raise ChgnetB200Error(f"self_energy_spectrum: q1 must be int32 [Q1], omega [F], p [Q1, {nb}, {nb}, {nb}], "
                                  f"temperatures [T] and gamma [T, {nb}, F]")
        work = torch.empty(max(1, se_scratch_doubles(nb, n_f, n_t)), dtype=torch.float64, device=freqs.device)
        self._call("chg_self_energy_spectrum", _p(freqs), nb, n1, n2, n3, _p(tetrahedra), int(target), _p(omega), n_f,
                   _p(q1), n_q1, _p(p), _p(temperatures), n_t, float(cutoff_thz), _p(work), work.numel(), _p(gamma))

    def coherence_conductivity(self, freqs, eigvecs, ddyn, set_id, heat_capacity, gamma, cutoff_thz, kappa):
        """kappa [T, 3, 3] fp64 += the unscaled Wigner coherence pair sum of the q of the call
        (``chg_coherence_conductivity``, DESIGN.md section 12.10): freqs [Q, n_band] THz (the Gamma acoustic modes
        already 0), eigvecs [Q, mode, n_band] complex128 (mode-major), ddyn [Q, 3, n_band, n_band] complex128 as
        ``dynamical_matrix_derivatives`` writes it, set_id [Q, n_band] int32 degenerate-set ids, heat_capacity (eV/K)
        and gamma (THz) [T, Q, n_band]; pairs of modes below cutoff_thz, with Gamma <= 0 or in one set are left out."""
        self._chk(freqs, eigvecs, ddyn, set_id, heat_capacity, gamma, kappa)
        f64, c128 = torch.float64, torch.complex128
        if (any(t.dtype != f64 for t in (freqs, heat_capacity, gamma, kappa)) or eigvecs.dtype != c128
                or ddyn.dtype != c128 or set_id.dtype != torch.int32):
            raise ChgnetB200Error("coherence_conductivity: eigvecs and ddyn must be complex128, set_id int32 and every "
                                  "other tensor float64")
        n_q, nb = freqs.shape
        n_t = gamma.shape[0]
        if (tuple(eigvecs.shape) != (n_q, nb, nb) or tuple(ddyn.shape) != (n_q, 3, nb, nb)
                or tuple(set_id.shape) != (n_q, nb) or tuple(heat_capacity.shape) != (n_t, n_q, nb)
                or tuple(gamma.shape) != (n_t, n_q, nb) or tuple(kappa.shape) != (n_t, 3, 3)):
            raise ChgnetB200Error(f"coherence_conductivity: freqs must be [Q, n_band], eigvecs [{n_q}, {nb}, {nb}], "
                                  f"ddyn [{n_q}, 3, {nb}, {nb}], set_id [{n_q}, {nb}], heat_capacity and gamma "
                                  f"[T, {n_q}, {nb}] and kappa [T, 3, 3]")
        work = torch.empty(max(1, coherence_scratch_doubles(n_q, nb, n_t)), dtype=f64, device=freqs.device)
        self._call("chg_coherence_conductivity", _p(freqs), _p(eigvecs), _p(ddyn), _p(set_id), _p(heat_capacity),
                   _p(gamma), n_q, nb, n_t, float(cutoff_thz), _p(work), work.numel(), _p(kappa))

    def isotope_scattering(self, freqs, mesh, tetrahedra, eigvecs, mass_variances, targets, omega, cutoff_thz, gamma):
        """gamma [Q, n_band] fp64 (overwritten) = the isotope scattering rates (half width, THz) of the targets' modes at
        w = omega [Q, n_band], before degenerate averaging (``chg_isotope_scattering``, DESIGN.md section 12.11):
        freqs [n1 n2 n3, n_band] THz and eigvecs [n1 n2 n3, mode, n_band] complex128 (mode-major) of the full
        Gamma-centred ``mesh``, tetrahedra [6, 4, 3] int32, mass_variances [n_band / 3] fp64, targets [Q] int32 mesh
        indices; vertex modes below cutoff_thz take no part, and w below cutoff_thz gives 0."""
        self._chk(freqs, tetrahedra, eigvecs, mass_variances, targets, omega, gamma)
        n1, n2, n3 = _mesh_args("isotope_scattering", mesh, freqs, tetrahedra,
                                "freqs, mass_variances, omega and gamma", (freqs, mass_variances, omega, gamma))
        n_q, nb = freqs.shape
        n_target = targets.shape[0]
        if (eigvecs.dtype != torch.complex128 or tuple(eigvecs.shape) != (n_q, nb, nb) or nb % 3
                or tuple(mass_variances.shape) != (nb // 3,) or targets.dtype != torch.int32 or targets.dim() != 1
                or tuple(omega.shape) != (n_target, nb) or tuple(gamma.shape) != (n_target, nb)):
            raise ChgnetB200Error(f"isotope_scattering: eigvecs must be complex128 [{n_q}, {nb}, {nb}], mass_variances "
                                  f"[{nb // 3}], targets int32 [Q], omega and gamma [Q, {nb}]")
        work = torch.empty(max(1, isotope_scratch_doubles(n_target, n_q, nb)), dtype=torch.float64, device=freqs.device)
        self._call("chg_isotope_scattering", _p(freqs), _p(eigvecs), nb, n1, n2, n3, _p(tetrahedra),
                   _p(mass_variances), nb // 3, _p(targets), n_target, _p(omega), float(cutoff_thz), _p(gamma),
                   _p(work), work.numel())

    def sample_displacements(self, evecs, amp, inv_sqrt_m, frac_ref, lattice, inv_lattice, seed, iteration,
                             first_sample, frac, u):
        """frac [M N, 3] fp32 and u [M, N, 3] fp64 (written): the thermal displacement samples first_sample ...
        first_sample + M - 1 of the supercell (``chg_sample_displacements``, DESIGN.md section 12.12): evecs
        [3N, 3N] fp64 row lam the unit mode vector, amp [3N], inv_sqrt_m [N], frac_ref [N, 3], lattice and inv_lattice
        [3, 3] fp64; the variates are a function of (seed, iteration, sample, mode) only."""
        self._chk(evecs, amp, inv_sqrt_m, frac_ref, lattice, inv_lattice, frac, u)
        n3 = evecs.shape[0]
        m = u.shape[0]
        if (any(t.dtype != torch.float64 for t in (evecs, amp, inv_sqrt_m, frac_ref, lattice, inv_lattice, u))
                or frac.dtype != torch.float32 or n3 % 3 or tuple(evecs.shape) != (n3, n3) or tuple(amp.shape) != (n3,)
                or tuple(inv_sqrt_m.shape) != (n3 // 3,) or tuple(frac_ref.shape) != (n3 // 3, 3)
                or tuple(lattice.shape) != (3, 3) or tuple(inv_lattice.shape) != (3, 3)
                or tuple(frac.shape) != (m * (n3 // 3), 3) or tuple(u.shape) != (m, n3 // 3, 3)):
            raise ChgnetB200Error(f"sample_displacements: frac must be float32 [M N, 3] and every other tensor float64: "
                                  f"evecs [3N, 3N], amp [3N], inv_sqrt_m [N], frac_ref [N, 3], lattice and "
                                  f"inv_lattice [3, 3], u [M, N, 3]")
        work = torch.empty(max(1, sampler_scratch_doubles(m, n3)), dtype=torch.float64, device=u.device)
        self._call("chg_sample_displacements", _p(evecs), _p(amp), n3, _p(inv_sqrt_m), _p(frac_ref), _p(lattice),
                   _p(inv_lattice), int(seed), int(iteration), int(first_sample), m, _p(work), work.numel(), _p(frac),
                   _p(u))

    def displacement_moments(self, u, force, f0, perm, acc):
        """acc [2 n_prim 9 N + 2] fp64 += the folded moments G_c, B, sum |dF|^2 and sum f0 . u of the samples u and
        force [M, N, 3] fp64 (``chg_displacement_moments``, DESIGN.md section 12.12): f0 [N, 3] fp64, perm [n_cells, N]
        int32 the supercell translations, n_prim = N / n_cells."""
        self._chk(u, force, f0, perm, acc)
        m, n = u.shape[0], u.shape[1]
        n_cells = perm.shape[0]
        if (any(t.dtype != torch.float64 for t in (u, force, f0, acc)) or perm.dtype != torch.int32 or n_cells < 1
                or n % n_cells or tuple(u.shape) != (m, n, 3) or tuple(force.shape) != (m, n, 3)
                or tuple(f0.shape) != (n, 3) or tuple(perm.shape) != (n_cells, n)
                or tuple(acc.shape) != (18 * (n // n_cells) * n + 2,)):
            raise ChgnetB200Error("displacement_moments: u and force must be float64 [M, N, 3], f0 [N, 3], perm int32 "
                                  "[n_cells, N] with n_cells dividing N, acc float64 [18 n_prim N + 2]")
        work = torch.empty(max(1, moments_scratch_doubles(m, n // n_cells, n)), dtype=torch.float64, device=u.device)
        self._call("chg_displacement_moments", _p(u), _p(force), _p(f0), _p(perm), n, n_cells, m, _p(work),
                   work.numel(), _p(acc))

    def atom_conv_tan(self, pcn_d, pe_d, wag, wag_d, center, nbr, d2u, save_pre, save_p, w2t, ln, msg_d, pre_d, p_d):
        self._chk(pcn_d, pe_d, wag, wag_d, center, nbr, d2u, save_pre, save_p, w2t, ln, msg_d, pre_d, p_d)
        self._call("chg_atom_conv_tan", _p(pcn_d), _p(pe_d), _p(wag), _p(wag_d), _p(center), _p(nbr), _p(d2u),
                   center.shape[0], _p(save_pre), _p(save_p), _p(w2t), _p(ln), _p(msg_d), _p(pre_d), _p(p_d))

    def atom_conv_bwd2(self, save_pre, save_p, pre_d, p_d, g_p_lam, wag, wag_d, center, d2u, lam_agg, bar_agg, w2, ln,
                       bar_pre, bar_w, u_out, g_ln):
        self._chk(save_pre, save_p, pre_d, p_d, g_p_lam, wag, wag_d, center, d2u, lam_agg, bar_agg, w2, ln, bar_pre,
                  bar_w, u_out, g_ln)
        self._call("chg_atom_conv_bwd2", _p(save_pre), _p(save_p), _p(pre_d), _p(p_d), _p(g_p_lam), _p(wag), _p(wag_d),
                   _p(center), _p(d2u), center.shape[0], _p(lam_agg), _p(bar_agg), _p(w2), _p(ln), _p(bar_pre), _p(bar_w),
                   _p(u_out), _p(g_ln))

    def bond_conv_tan(self, pij_d, px_d, pa_d, wbg, wbg_d, ang_atom, ang_i, ang_j, save_pre, save_p, w2t, ln, upd_d,
                      pre_d, p_d):
        self._chk(pij_d, px_d, pa_d, wbg, wbg_d, ang_atom, ang_i, ang_j, save_pre, save_p, w2t, ln, upd_d, pre_d, p_d)
        self._call("chg_bond_conv_tan", _p(pij_d), _p(px_d), _p(pa_d), _p(wbg), _p(wbg_d), _p(ang_atom), _p(ang_i),
                   _p(ang_j), ang_i.shape[0], _p(save_pre), _p(save_p), _p(w2t), _p(ln), _p(upd_d), _p(pre_d), _p(p_d))

    def bond_conv_bwd2(self, save_pre, save_p, pre_d, p_d, g_p_lam, wbg, wbg_d, ang_i, ang_j, lam_agg, bar_agg, w2, ln,
                       bar_pre, bar_wi, bar_wj, u_out, g_ln):
        self._chk(save_pre, save_p, pre_d, p_d, g_p_lam, wbg, wbg_d, ang_i, ang_j, lam_agg, bar_agg, w2, ln, bar_pre,
                  bar_wi, bar_wj, u_out, g_ln)
        self._call("chg_bond_conv_bwd2", _p(save_pre), _p(save_p), _p(pre_d), _p(p_d), _p(g_p_lam), _p(wbg), _p(wbg_d),
                   _p(ang_i), _p(ang_j), ang_i.shape[0], _p(lam_agg), _p(bar_agg), _p(w2), _p(ln), _p(bar_pre),
                   _p(bar_wi), _p(bar_wj), _p(u_out), _p(g_ln))

    def angle_update_tan(self, pij_d, px_d, pa_d, ang_d, ang_atom, ang_i, ang_j, save_p, ln, ang_new_d, p_d):
        self._chk(pij_d, px_d, pa_d, ang_d, ang_atom, ang_i, ang_j, save_p, ln, ang_new_d, p_d)
        self._call("chg_angle_update_tan", _p(pij_d), _p(px_d), _p(pa_d), _p(ang_d), _p(ang_atom), _p(ang_i), _p(ang_j),
                   ang_i.shape[0], _p(save_p), _p(ln), _p(ang_new_d), _p(p_d))

    def angle_update_bwd2(self, save_p, p_d, lam_ang, bar_ang, ln, bar_pre, g_ln):
        self._chk(save_p, p_d, lam_ang, bar_ang, ln, bar_pre, g_ln)
        self._call("chg_angle_update_bwd2", _p(save_p), _p(p_d), _p(lam_ang), _p(bar_ang), save_p.shape[0], _p(ln),
                   _p(bar_pre), _p(g_ln))

    def readout_bwd2(self, x, xd, ln, mlp_wt, mlp_w, mlp_b, w_last, seed, bar_x, h_all, hd_all, gz_all, zbar_all,
                     g_h0, hbar0, xhat, xhatd):
        self._chk(x, xd, ln, mlp_wt, mlp_w, mlp_b, w_last, seed, bar_x, h_all, hd_all, gz_all, zbar_all, g_h0, hbar0,
                  xhat, xhatd)
        self._call("chg_readout_bwd2", _p(x), _p(xd), x.shape[0], _p(ln), _p(mlp_wt), _p(mlp_w), _p(mlp_b),
                   mlp_wt.shape[0], _p(w_last), _p(seed), _p(bar_x), _p(h_all), _p(hd_all), _p(gz_all), _p(zbar_all),
                   _p(g_h0), _p(hbar0), _p(xhat), _p(xhatd))

    def adam_step(self, p, g, m, v, lr, beta1, beta2, eps, weight_decay, step):
        self._chk(p, g, m, v)
        self._call("chg_adam_step", _p(p), _p(g), _p(m), _p(v), p.numel(), float(lr), float(beta1), float(beta2),
                   float(eps), float(weight_decay), int(step))

    def readout(self, x, z, owner, ln, mlp_wt, mlp_w, mlp_b, w_last, b_last, atom_ref, site_e, h_out, e_graph,
                e_ref, g_x):
        self._chk(x, z, owner, ln, mlp_wt, mlp_w, mlp_b, w_last, atom_ref, site_e, h_out, e_graph, e_ref, g_x)
        self._call("chg_readout", _p(x), _p(z), _p(owner), x.shape[0], _p(ln), _p(mlp_wt), _p(mlp_w), _p(mlp_b),
                   mlp_wt.shape[0], _p(w_last), float(b_last), _p(atom_ref), _p(site_e), _p(h_out), _p(e_graph),
                   _p(e_ref), _p(g_x))

    def magmom(self, x, w, b, m):
        self._chk(x, w, m)
        self._call("chg_magmom", _p(x), x.shape[0], _p(w), float(b), _p(m))

    def force_virial(self, rvec, dist, rhat, g_rhat, g_dist, d2u, u2d, center, nbr, owner, force, virial):
        self._chk(rvec, dist, rhat, g_rhat, g_dist, d2u, u2d, center, nbr, owner, force, virial)
        self._call("chg_force_virial", _p(rvec), _p(dist), _p(rhat), _p(g_rhat), _p(g_dist), _p(d2u), _p(u2d),
                   _p(center), _p(nbr), _p(owner), center.shape[0], _p(force), _p(virial))
