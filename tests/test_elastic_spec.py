"""CPU: strain second derivatives of the kernel schedule (Engine.second_derivatives), with the torch kernel
specifications injected in fp64, against autograd through the oracle's create_graph=True stress and forces
(oracle/elastic.py); the LiMnO2 clamped-ion, internal-strain and relaxed-ion tensors assembled as
CHGNet.predict_elastic_tensor assembles them; the oracle strain blocks against the ones the live reference computed
(tests/golden/chgnet_0.3.0_elastic.npz)."""
import os

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import EV_A3_TO_GPA, Engine
from chgnet_b200.model import _VOIGT_DIRECTIONS, _relax_ions
from chgnet_b200.weights import pack_weights
from oracle.elastic import ElasticSpecKernels, oracle_elastic, oracle_strain_blocks
from oracle.hessian import oracle_hvp

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "chgnet_0.3.0_elastic.npz")


def spec_engine(weights):
    sd = {k: torch.as_tensor(np.asarray(v)).double() for k, v in weights.items()}
    return Engine(pack_weights(sd, None, device="cpu", dtype=torch.float64), ElasticSpecKernels())


def spec_batch(graphs, compact=True):
    b = build_batch(graphs, "cpu", compact_bonds=compact)
    b.frac, b.lattice, b.image = b.frac.double(), b.lattice.double(), b.image.double()
    return b


def oracle_second_derivatives(weights, graphs, v, w):
    """(H v + Lambda W per atom, Lambda^T v + D W per graph) from the oracle's double backward."""
    hv = oracle_hvp(weights, graphs, v)
    per_atom, per_graph, off = [], [], 0
    for k, g in enumerate(graphs):
        n = g.atomic_number.shape[0]
        D, lam = oracle_strain_blocks(weights, g)
        lam = torch.as_tensor(lam).view(n, 3, 3, 3)
        per_atom.append(hv[off : off + n] + torch.einsum("mbij,ij->mb", lam, w[k]))
        per_graph.append(torch.einsum("mbij,mb->ij", lam, v[off : off + n]) + torch.einsum("ijkl,kl->ij", torch.as_tensor(D), w[k]))
        off += n
    return torch.cat(per_atom), torch.stack(per_graph)


def _check(got, want, rel=1e-6):
    for g, t in zip(got, want):
        scale = float(t.abs().max())
        assert scale > 1e-3
        assert float((g - t).abs().max()) <= rel * scale, (float((g - t).abs().max()), scale)


@pytest.mark.parametrize("compact", [True, False])
def test_second_derivatives_match_oracle_double_backward(weights030, compact):
    graphs = graphgen.random_graphs(3, 6, 10, 8800)
    sizes = [g.atomic_number.shape[0] for g in graphs]
    gen = torch.Generator().manual_seed(21)
    v = torch.randn(sum(sizes), 3, generator=gen, dtype=torch.float64)
    v[sizes[0] : sizes[0] + sizes[1]] = 0.0  # graph 1: a strain direction only
    w = torch.randn(3, 3, 3, generator=gen, dtype=torch.float64)
    w[0] = 0.0  # graph 0: a position direction only; graph 2: both
    want = oracle_second_derivatives(weights030, graphs, v, w)
    got = spec_engine(weights030).second_derivatives(spec_batch(graphs, compact), v, w)
    assert got[0].shape == (sum(sizes), 3) and got[1].shape == (3, 3, 3) and got[1].dtype == torch.float64
    _check(got, want)


def test_second_derivatives_without_angles_and_with_isolated_atom(weights030):
    g_noang = graphgen.make_crystal_graph([3, 8], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 5.5)
    g_iso = graphgen.make_crystal_graph([3], np.zeros((1, 3)), np.eye(3) * 20.0)
    graphs = [g_iso, g_noang]
    assert len(g_noang.bond_graph) == 0 and len(g_iso.atom_graph) == 0
    gen = torch.Generator().manual_seed(22)
    v = torch.randn(3, 3, generator=gen, dtype=torch.float64)
    w = torch.randn(2, 3, 3, generator=gen, dtype=torch.float64)
    want = oracle_second_derivatives(weights030, graphs, v, w)
    got = spec_engine(weights030).second_derivatives(spec_batch(graphs), v, w)
    assert float(got[0][0].abs().max()) == 0.0 and float(got[1][0].abs().max()) == 0.0  # the isolated atom feels nothing
    assert torch.isfinite(got[0]).all() and torch.isfinite(got[1]).all()
    _check((got[0][1:], got[1][1:]), (want[0][1:], want[1][1:]))


def test_zero_strain_direction_is_the_hessian_vector_product(weights030):
    graphs = graphgen.random_graphs(2, 6, 9, 8801)
    n = sum(g.atomic_number.shape[0] for g in graphs)
    v = torch.randn(n, 3, generator=torch.Generator().manual_seed(23), dtype=torch.float64)
    eng = spec_engine(weights030)
    hv, _ = eng.second_derivatives(spec_batch(graphs), v, torch.zeros(2, 3, 3, dtype=torch.float64))
    want = eng.hessian_vector_products(spec_batch(graphs), v)
    assert float((hv - want).abs().max()) <= 1e-12 * float(want.abs().max())


def spec_elastic(eng, graph, chunk=12):
    """predict_elastic_tensor's assembly, on the fp64 specifications: 6 Voigt strain columns, then 3N position columns."""
    n = graph.atomic_number.shape[0]
    k_all = 6 + 3 * n
    v = np.zeros((k_all, 3 * n))
    v[6:] = np.eye(3 * n)
    w = np.zeros((k_all, 3, 3))
    w[:6] = _VOIGT_DIRECTIONS
    per_atom, per_graph = [], []
    for s in range(0, k_all, chunk):
        k = min(chunk, k_all - s)
        a, g = eng.second_derivatives(spec_batch([graph] * k), torch.as_tensor(v[s : s + k]).view(k * n, 3),
                                      torch.as_tensor(w[s : s + k]))
        per_atom.append(a.view(k, 3 * n).numpy())
        per_graph.append(g.numpy())
    per_atom, per_graph = np.concatenate(per_atom), np.concatenate(per_graph)
    scale = EV_A3_TO_GPA / abs(float(np.linalg.det(graph.lattice.double().numpy())))
    clamped = scale * np.einsum("aij,bij->ab", _VOIGT_DIRECTIONS, per_graph[:6])
    lam = per_atom[:6].T.copy()
    h = per_atom[6:].T.copy()
    with pytest.warns(RuntimeWarning, match="1 unstable mode"):
        relaxed, unstable = _relax_ions(clamped, lam, h, scale)
    lam_from_positions = np.einsum("aij,cij->ca", _VOIGT_DIRECTIONS, per_graph[6:])
    return dict(clamped_ion=clamped, internal_strain=lam, relaxed_ion=relaxed, unstable_modes=unstable, hessian=h,
                lam_from_positions=lam_from_positions)


@pytest.fixture(scope="module")
def limno2_elastic(weights030, limno2_graph):
    return spec_elastic(spec_engine(weights030), limno2_graph), oracle_elastic(weights030, limno2_graph)


def test_limno2_elastic_matches_oracle(limno2_elastic):
    got, want = limno2_elastic
    for key in ("clamped_ion", "internal_strain", "relaxed_ion", "hessian"):
        scale = np.abs(want[key]).max()
        assert np.abs(got[key] - want[key]).max() <= 1e-9 * scale, key
    assert got["unstable_modes"] == want["unstable_modes"] == 1
    c = got["clamped_ion"]
    assert np.abs(c - c.T).max() <= 1e-10 * np.abs(c).max()
    assert np.abs(got["internal_strain"].reshape(-1, 3, 6).sum(axis=0)).max() <= 1e-9 * np.abs(got["internal_strain"]).max()
    # the orthorhombic cell's tensors, to the 0.1 GPa they are quoted at
    diag_c = [369.7, 112.4, 281.6, 41.4, 75.4, 39.9]
    off_c = [c[0, 1], c[0, 2], c[1, 2]]
    assert np.abs(np.diag(c) - diag_c).max() < 0.06 and np.abs(np.array(off_c) - [64.5, 152.0, 65.4]).max() < 0.06
    r = got["relaxed_ion"]
    assert np.abs(np.diag(r) - [300.0, 102.6, 135.0, 34.6, 28.7, 39.9]).max() < 0.06
    assert np.abs(np.array([r[0, 1], r[0, 2], r[1, 2]]) - [53.4, 51.1, 47.5]).max() < 0.06


def test_internal_strain_from_strain_and_position_columns_agree(limno2_elastic):
    got, _ = limno2_elastic
    lam = got["internal_strain"]
    assert np.abs(got["lam_from_positions"] - lam).max() <= 1e-9 * np.abs(lam).max()


def test_relax_ions_isolated_atom_and_flat_energy():
    c = np.arange(36.0).reshape(6, 6)
    relaxed, unstable = _relax_ions(c, np.zeros((3, 6)), np.zeros((3, 3)), 1.0)  # one atom
    assert unstable == 0 and np.array_equal(relaxed, c)
    relaxed, unstable = _relax_ions(c, np.zeros((6, 6)), np.zeros((6, 6)), 1.0)  # no bonds: H = 0
    assert unstable == 0 and np.array_equal(relaxed, c)


def test_oracle_strain_blocks_match_live_reference(weights030, limno2_graph):
    with np.load(GOLDEN) as f:
        gold = {k: f[k] for k in f.files}
    cases = [("limno2", limno2_graph)]
    cases.append(("random", graphgen.make_crystal_graph(gold["random.z"], gold["random.frac"], gold["random.lattice"])))
    for name, g in cases:
        D, lam = oracle_strain_blocks(weights030, g)
        for key, got in (("strain_strain", D), ("internal_strain", lam)):
            want = gold[f"{name}.{key}"]
            tol = float(gold[f"{name}.rtol"]) * np.abs(want).max()
            assert np.abs(got - want).max() <= tol, (name, key, np.abs(got - want).max(), tol, str(gold["dtype"]))
