"""CPU: Hessian-vector products of the kernel schedule (Engine.hessian_vector_products), with the torch kernel
specifications injected in fp64, against autograd through the oracle's create_graph=True forces (oracle/hessian.py); the oracle
Hessian of LiMnO2 against the one the live reference computed (tests/golden/chgnet_0.3.0_hessian.npz)."""
import os

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights
from oracle.hessian import HessianSpecKernels, oracle_hessian, oracle_hvp
from oracle.kernel_specs import SpecKernels

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "chgnet_0.3.0_hessian.npz")


def spec_engine(weights):
    sd = {k: torch.as_tensor(np.asarray(v)).double() for k, v in weights.items()}
    return Engine(pack_weights(sd, None, device="cpu", dtype=torch.float64), HessianSpecKernels())


def spec_batch(graphs, compact=True):
    b = build_batch(graphs, "cpu", compact_bonds=compact)
    b.frac, b.lattice, b.image = b.frac.double(), b.lattice.double(), b.image.double()
    return b


def spec_hessian(eng, graph, chunk=12):
    n = graph.atomic_number.shape[0]
    cols = []
    for s in range(0, 3 * n, chunk):
        k = min(chunk, 3 * n - s)
        v = torch.zeros(k, n * 3, dtype=torch.float64)
        v[torch.arange(k), torch.arange(s, s + k)] = 1.0
        hv = eng.hessian_vector_products(spec_batch([graph] * k), v.view(k * n, 3))
        cols.append(hv.view(k, 3 * n))
    return torch.cat(cols).T.numpy()  # column c = H e_c


@pytest.mark.parametrize("compact", [True, False])
def test_hvp_matches_oracle_double_backward(weights030, compact):
    graphs = graphgen.random_graphs(3, 6, 10, 8700)
    n_atoms = sum(g.atomic_number.shape[0] for g in graphs)
    v = torch.randn(n_atoms, 3, generator=torch.Generator().manual_seed(11), dtype=torch.float64)
    want = oracle_hvp(weights030, graphs, v)
    got = spec_engine(weights030).hessian_vector_products(spec_batch(graphs, compact), v)
    scale = float(want.abs().max())
    assert scale > 1e-3
    assert float((got - want).abs().max()) <= 1e-6 * scale


def test_hvp_without_angles_and_with_isolated_atom(weights030):
    g_noang = graphgen.make_crystal_graph([3, 8], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 5.5)
    g_iso = graphgen.make_crystal_graph([3], np.zeros((1, 3)), np.eye(3) * 20.0)
    graphs = [g_iso, g_noang]
    assert len(g_noang.bond_graph) == 0 and len(g_iso.atom_graph) == 0
    v = torch.randn(3, 3, generator=torch.Generator().manual_seed(12), dtype=torch.float64)
    want = oracle_hvp(weights030, graphs, v)
    got = spec_engine(weights030).hessian_vector_products(spec_batch(graphs), v)
    assert float(got[0].abs().max()) == 0.0  # the isolated atom feels nothing
    assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max())


@pytest.fixture(scope="module")
def limno2_hessians(weights030, limno2_graph):
    return spec_hessian(spec_engine(weights030), limno2_graph), oracle_hessian(weights030, limno2_graph)


def test_limno2_hessian_matches_oracle(limno2_graph, limno2_hessians):
    got, want = limno2_hessians
    # the cell has exactly collinear bond pairs: the (1 - 1e-6) regularised acos is at its stiffest there
    b = spec_batch([limno2_graph])
    rvec, dist, rhat = torch.empty(b.n_edges, 3, dtype=torch.float64), torch.empty(b.n_edges, dtype=torch.float64), \
        torch.empty(b.n_edges, 3, dtype=torch.float64)
    SpecKernels().edge_geometry(b.frac, b.lattice, b.owner, b.center, b.nbr, b.image, rvec, dist, rhat)
    cos = (rhat[b.ang_di.long()] * rhat[b.ang_dj.long()]).sum(dim=1)
    assert int((cos < -1 + 1e-12).sum()) == 16
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 1e-6 * scale
    assert np.abs(got - got.T).max() <= 1e-7 * scale
    n = got.shape[0] // 3
    acoustic = got.reshape(3 * n, n, 3).sum(axis=1)  # sum_j H[ia, jb]: a rigid translation costs nothing
    assert np.abs(acoustic).max() <= 1e-9 * scale


def test_oracle_hessian_matches_live_reference(weights030, limno2_graph, limno2_hessians):
    with np.load(GOLDEN) as f:
        gold = {k: f[k] for k in f.files}
    want = gold["limno2.hessian"]
    got = limno2_hessians[1]
    tol = float(gold["limno2.rtol"]) * np.abs(want).max()
    assert np.abs(got - want).max() <= tol, (np.abs(got - want).max(), tol, str(gold["dtype"]))
    z, frac, lat = gold["random.z"], gold["random.frac"], gold["random.lattice"]
    g = graphgen.make_crystal_graph(z, frac, lat)
    want = gold["random.hessian"]
    got = oracle_hessian(weights030, g)
    assert np.abs(got - want).max() <= float(gold["random.rtol"]) * np.abs(want).max()
