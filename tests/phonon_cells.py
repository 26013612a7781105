"""Crystals for the phonon tests: spring crystals whose bands are known in closed form, LiMnO2 2x1x1 with the fp64
oracle's force constants, and LiMnO2 2x2x2 with the device force constants of the 0.3.0 weights."""
import os

import numpy as np

from chgnet_b200 import graphgen
from chgnet_b200.phonons import THZ_PER_SQRT_EV_A2_AMU, Phonons, make_supercell
from oracle.phonons import PhononSpecKernels, oracle_compact_fcs

GOLD = os.path.join(os.path.dirname(__file__), "golden")
# fcc Cu, one atom per rhombohedral primitive cell
CU = (np.array([29]), np.zeros((1, 3)), 1.805 * (np.ones((3, 3)) - np.eye(3)))
# spring crystals: lattice constant (A), spring constant (eV/A^2) and atomic number
A, K, Z = 2.7, 3.0, 13


def spec_phonons(fc, sc) -> Phonons:
    """``Phonons`` of the force constants ``fc`` on the supercell ``sc``, on the host with the fp64 specifications of
    the kernels."""
    return Phonons(fc, sc, device="cpu", kernels=PhononSpecKernels())


def springs(m, ks=(K, K, K), a=(A, A, A)):
    """One atom per cell of the orthorhombic lattice diag(a), nearest-neighbour central springs ks along the axes
    (three independent 1D chains), on the supercell ``m``.  Returns the spec-path ``Phonons`` and nu_max [3] (THz):
    branch c has nu_c(q) = nu_max,c |sin pi q_c|."""
    sc = make_supercell([Z], np.zeros((1, 3)), np.diag(np.asarray(a, dtype=np.float64)), m)
    inv = np.linalg.inv(sc.lattice)
    fc = np.zeros((1, len(sc.z), 3, 3))
    for c in range(3):
        for sgn in (1, -1):
            x = ((sgn * a[c] * np.eye(3)[c]) @ inv) % 1.0  # supercell fractional position of the neighbour
            j = int(np.argmin(np.abs((sc.frac - x + 0.5) % 1.0 - 0.5).sum(1)))
            fc[0, j, c, c] -= ks[c]
        fc[0, 0, c, c] += 2 * ks[c]
    ph = spec_phonons(fc, sc)
    return ph, THZ_PER_SQRT_EV_A2_AMU * np.sqrt(4 * np.asarray(ks) / ph.masses[0])


def limno2_211(weights):
    """LiMnO2 2x1x1: the supercell, its graph and the oracle's compact force constants for ``weights``."""
    sc = make_supercell(*graphgen.limno2_structure(), [2, 1, 1])
    g = graphgen.make_crystal_graph(sc.z, sc.frac, sc.lattice)
    return sc, g, oracle_compact_fcs(weights, g, sc.p2s)


def limno2_211_spec(weights) -> Phonons:
    """The spec-path ``Phonons`` of ``limno2_211``."""
    sc, _, fc = limno2_211(weights)
    return spec_phonons(fc, sc)


def model030():
    """The 0.3.0 model on the device."""
    from chgnet_b200.model import CHGNet

    return CHGNet.from_file(os.path.join(GOLD, "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")


def limno2_222(model) -> Phonons:
    """LiMnO2 2x2x2 ``Phonons`` from the device force constants of ``model``."""
    return model.phonons(graphgen.limno2_structure(), [2, 2, 2])
