"""The architecture variants of tests/test_architectures_spec.py and tests/test_architectures_gpu.py: one option of the
0.3.0 shape changed per variant, their weights, and cells built with their cutoffs."""
from __future__ import annotations

import functools

import numpy as np
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch

# the CHGNet constructor's keywords of each variant
VARIANTS = {
    "basis-1-1": dict(num_radial=1, num_angular=1),
    "basis-16-3": dict(num_radial=16, num_angular=3),
    "basis-32-31": dict(num_radial=32, num_angular=31),
    "conv-1": dict(n_conv=1),
    "conv-2": dict(n_conv=2),
    "conv-5": dict(n_conv=5),
    "conv-8": dict(n_conv=8),
    "readout-int": dict(mlp_hidden_dims=64),
    "readout-1": dict(mlp_hidden_dims=[64]),
    "readout-4": dict(mlp_hidden_dims=[64] * 4),
    "ln-gmlp-only": dict(readout_norm=None),
    "ln-readout-only": dict(gMLP_norm=None),
    "envelope-p1": dict(cutoff_coeff=1),
    "envelope-p3": dict(cutoff_coeff=3),
    "cutoffs-4.5-2.5": dict(atom_graph_cutoff=4.5, bond_graph_cutoff=2.5),
    "cutoffs-4-4": dict(atom_graph_cutoff=4.0, bond_graph_cutoff=4.0),
    "extensive": dict(is_intensive=False),
    "frozen-rbf": dict(learnable_rbf=False),
}
_ORACLE_KEYS = ("num_radial", "num_angular", "n_conv", "cutoff_coeff", "gMLP_norm", "readout_norm", "is_intensive")


def _rescaled(sd: dict, seed: int) -> dict[str, np.ndarray]:
    """Seeded values for the constructor's state_dict, scaled like ``oracle.chgnet_oracle.random_weights``.

    The constructor's initialisation (zero biases, unit LayerNorms, U(+-1/sqrt(in)) weights) gives forces of ~1e-4 eV/A,
    under the end-to-end tolerances; these weights give forces and stresses of order one."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, v in sd.items():
        v = v.detach().cpu().numpy()
        if k.startswith("composition_model."):
            out[k] = v
        elif k.endswith("frequencies"):
            out[k] = (v * rng.uniform(0.9, 1.1, v.shape)).astype(np.float32)
        elif (".bn" in k or k.startswith("readout_norm.")) and k.endswith(".weight"):
            out[k] = (1.0 + 0.1 * rng.standard_normal(v.shape)).astype(np.float32)
        elif k.endswith(".bias"):
            out[k] = (0.1 * rng.standard_normal(v.shape)).astype(np.float32)
        elif k == "atom_embedding.embedding.weight":
            out[k] = rng.standard_normal(v.shape).astype(np.float32)
        else:
            scale = 0.3 if ".mlp_out." in k else 1.0
            out[k] = (rng.standard_normal(v.shape) * scale / np.sqrt(v.shape[1])).astype(np.float32)
    return out


@functools.lru_cache(maxsize=None)
def architecture(variant: str):
    """(weights as numpy arrays, oracle args, model_args) of a variant: the state_dict of a seeded
    ``CHGNet(**VARIANTS[variant])`` with its values re-drawn by ``_rescaled``."""
    from chgnet_b200.model import CHGNet

    seed = sum(map(ord, variant))
    torch.manual_seed(seed)
    model = CHGNet(**VARIANTS[variant])
    w = _rescaled(model.state_dict(), seed)
    a = model.model_args
    args = {k: a[k] for k in _ORACLE_KEYS}
    args["atom_graph_cutoff"], args["bond_graph_cutoff"] = float(a["atom_graph_cutoff"]), float(a["bond_graph_cutoff"])
    return w, args, dict(a)


def new_model(variant: str, device=None):
    """a CHGNet of the variant holding the weights of ``architecture(variant)``"""
    from chgnet_b200.model import CHGNet

    w, _, _ = architecture(variant)
    model = CHGNet(**VARIANTS[variant])
    model.load_state_dict({k: torch.as_tensor(v) for k, v in w.items()})
    return model if device is None else model.to(device)


def trainable_names(variant: str) -> set[str]:
    w, _, _ = architecture(variant)
    frozen = {"composition_model.fc.weight"}
    if not VARIANTS[variant].get("learnable_rbf", True):
        frozen |= {k for k in w if k.endswith("frequencies")}
    return set(w) - frozen


def cutoffs(variant: str) -> dict:
    a = VARIANTS[variant]
    return dict(atom_graph_cutoff=float(a.get("atom_graph_cutoff", 6.0)), bond_graph_cutoff=float(a.get("bond_graph_cutoff", 3.0)))


def cells(variant: str, seed: int = 9300, n: int = 3, n_lo: int = 6, n_hi: int = 12):
    """``n`` random cells with the variant's cutoffs, a dimer (one bond per atom: edges, no angles) and an isolated atom"""
    cut = cutoffs(variant)
    rand = graphgen.random_graphs(n, n_lo, n_hi, seed, **cut)
    dimer = graphgen.make_crystal_graph([3, 8], [[0.0, 0.0, 0.0], [0.12, 0.0, 0.0]], 15.0 * np.eye(3), **cut)
    iso = graphgen.make_crystal_graph([26], np.zeros((1, 3)), 20.0 * np.eye(3), **cut)
    assert len(dimer.atom_graph) == 2 and len(dimer.bond_graph) == 0 and len(iso.atom_graph) == 0
    assert all(len(g.bond_graph) > 0 for g in rand)
    return [rand[0], dimer, iso, *rand[1:]]


def fp64_batch(graphs, compact=True):
    """a host batch whose geometry inputs are fp64 (fp64 truth needs fp64 coordinates)"""
    b = build_batch(graphs, "cpu", compact_bonds=compact)
    b.image = b.image.double()
    b.frac = torch.cat([g.atom_frac_coord.detach().double() for g in graphs])
    b.lattice = torch.stack([g.lattice.detach().double().reshape(9) for g in graphs])
    L = b.lattice.view(-1, 3, 3)
    b.volume = (L[:, 0] * torch.linalg.cross(L[:, 1], L[:, 2])).sum(dim=1)
    return b
