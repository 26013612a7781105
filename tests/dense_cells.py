"""High-coordination cells for the tests: segments longer than one 128-row tile.

Within the 6 A atom-graph cutoff rattled diamond has 158 edges per atom, and the simple cubic H/Li cell at 1.1 A
(a 3.3 A box, thinner than the cutoff) has about 700 edges and 6 800 angles per atom.  The batch puts them between a
random cell and an edgeless H2 box, so ragged and empty segments stay in."""
import numpy as np

from chgnet_b200 import graphgen

DIAMOND_A = 3.567  # conventional cubic cell of diamond, A
_DIAMOND_FRAC = np.array([[0, 0, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [0.5, 0.5, 0],
                          [0.25, 0.25, 0.25], [0.25, 0.75, 0.75], [0.75, 0.25, 0.75], [0.75, 0.75, 0.25]])


def _supercell(frac, lattice, reps, rattle, seed):
    cells = np.array(np.meshgrid(*[range(r) for r in reps], indexing="ij")).reshape(3, -1).T
    frac = ((frac[None] + cells[:, None]) / np.array(reps)).reshape(-1, 3)
    lattice = lattice * np.array(reps)[:, None]
    cart = frac @ lattice + np.random.default_rng(seed).normal(0.0, rattle, size=frac.shape)
    return cart @ np.linalg.inv(lattice), lattice


def diamond(reps=(2, 2, 2), rattle=0.03, seed=7):
    """Carbon diamond, ``reps`` conventional cells, Gaussian displacements of ``rattle`` A."""
    frac, lat = _supercell(_DIAMOND_FRAC, DIAMOND_A * np.eye(3), reps, rattle, seed)
    return np.full(len(frac), 6), frac, lat


def simple_cubic_hli(reps=(3, 3, 3), a=1.1, rattle=0.05, seed=8):
    """Simple cubic lattice of spacing ``a`` A with H and Li alternating, Gaussian displacements of ``rattle`` A.
    Unphysically dense: only the kernels' indexing is checked on it, not its energies."""
    frac, lat = _supercell(np.zeros((1, 3)), a * np.eye(3), reps, rattle, seed)
    ijk = np.rint(frac * np.array(reps)).astype(int)
    return np.where(ijk.sum(axis=1) % 2 == 0, 1, 3), frac, lat


def dense_graphs(**cut):
    """The high-coordination batch: a random cell, diamond, the edgeless H2 box and the simple cubic H/Li cell."""
    h2 = graphgen.make_crystal_graph([1, 1], [[0.0, 0.0, 0.0], [0.5, 0.5, 0.5]], 20.0 * np.eye(3), graph_id="h2", **cut)
    return [graphgen.random_graphs(1, 20, 40, 9910, **cut)[0],
            graphgen.make_crystal_graph(*diamond(), graph_id="diamond", **cut), h2,
            graphgen.make_crystal_graph(*simple_cubic_hli(), graph_id="sc-hli", **cut)]
