"""-m gpu: the device graph builder (csrc/graph_device.cu, SURVEY.md §8 row f1) against the host builders.

Integer outputs must be BIT-IDENTICAL to ``graphgen.build_graph_arrays`` (the numpy restatement pinned against the
reference's ``Graph`` class) and to the host C++ builder: atom_graph, neighbor_image, directed2undirected,
undirected2directed, bond_graph - on the cases of the reference's own graph tests (LiMnO2 384 / 744 / 192 at cutoffs
5 / 3, 672 / 744 / 336 at 6 / 3, the 2 x 2 x 6 supercell's 9216 / 17856 / 4608: reference
tests/test_crystal_graph.py:22-42, 256-278), random cells, cells thinner than the cutoff, fractional coordinates outside
[0, 1), isolated atoms, an empty bond graph - and the model must give the same answer through either path."""
import dense_cells
import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def builder():
    from chgnet_b200.graph_device import DeviceGraphBuilder

    return DeviceGraphBuilder("cuda", 6.0, 3.0)


def _host(z, frac, lat, r_atom, r_bond):
    c, n, img, d = graphgen.neighbor_list(frac, lat, r_atom)
    ag, d2u, u2d, bg = graphgen.build_graph_arrays(c, n, img, d, r_bond)
    return ag, img, d2u, u2d, bg


def _check(z, frac, lat, r_atom=6.0, r_bond=3.0):
    from chgnet_b200.graph_device import DeviceGraphBuilder, crystal_graph_from_device

    b = DeviceGraphBuilder("cuda", r_atom, r_bond)
    g = crystal_graph_from_device(b, z, frac, lat)
    ag, img, d2u, u2d, bg = _host(z, np.asarray(frac, float), np.asarray(lat, float), r_atom, r_bond)
    assert g.atom_graph.shape == (len(ag), 2) and g.bond_graph.shape == (len(bg), 5), (g.atom_graph.shape, len(ag), g.bond_graph.shape, len(bg))
    assert np.array_equal(g.atom_graph.numpy(), ag)
    assert np.array_equal(g.neighbor_image.numpy().astype(np.int64), np.asarray(img).reshape(-1, 3))
    assert np.array_equal(g.directed2undirected.numpy(), d2u) and np.array_equal(g.undirected2directed.numpy(), u2d)
    assert np.array_equal(g.bond_graph.numpy(), bg)
    return g


def test_limno2_counts_of_the_reference_tests():
    z, frac, lat = graphgen.limno2_structure()
    g = _check(z, frac, lat, 5.0, 3.0)
    assert (len(g.atom_graph), len(g.bond_graph), len(g.undirected2directed)) == (384, 744, 192)
    g = _check(z, frac, lat, 6.0, 3.0)
    assert (len(g.atom_graph), len(g.bond_graph), len(g.undirected2directed)) == (672, 744, 336)
    z, frac, lat = graphgen.limno2_structure((2, 2, 6))
    g = _check(z, frac, lat, 5.0, 3.0)
    assert (len(g.atom_graph), len(g.bond_graph), len(g.undirected2directed)) == (9216, 17856, 4608)


@pytest.mark.parametrize("seed,n", [(9700, 8), (9701, 23), (9702, 57), (9703, 120)])
def test_random_cells(seed, n):
    z, frac, lat = graphgen.random_structure(n, seed)
    _check(z, frac, lat)
    _check(z, frac, lat, 5.0, 3.0)


def test_edge_cases():
    # fractional coordinates outside [0, 1) and a triclinic cell thinner than the cutoff along one axis
    z, frac, lat = graphgen.random_structure(10, 9710)
    _check(z, frac + np.array([1.0, -2.0, 0.5]), lat)
    thin = np.array([[2.2, 0.0, 0.0], [0.7, 7.5, 0.0], [0.3, -0.9, 9.0]])
    _check([3, 8, 25], np.array([[0.1, 0.2, 0.3], [0.6, 0.7, 0.1], [0.4, 0.1, 0.8]]), thin)
    # every atom isolated (no edges at all), and edges but an empty bond graph
    g = _check([1, 1], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 20.0)
    assert len(g.atom_graph) == 0 and len(g.bond_graph) == 0
    g = _check([3, 8], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 5.5)
    assert len(g.atom_graph) > 0 and len(g.bond_graph) == 0
    # a single atom whose only neighbours are its own images
    _check([26], np.zeros((1, 3)), np.eye(3) * 2.5)
    # hundreds of neighbours per centre: rattled diamond (158 edges per atom), and the 3.3 A simple cubic H/Li cell,
    # thinner than the cutoff, with about 700 edges and 6 800 angles per atom
    g = _check(*dense_cells.diamond())
    assert int(np.bincount(g.atom_graph[:, 0].numpy()).max()) > 128
    g = _check(*dense_cells.simple_cubic_hli())
    assert int(np.bincount(g.atom_graph[:, 0].numpy()).max()) > 512 and int(np.bincount(g.bond_graph[:, 0].numpy()).max()) > 4096


def test_c4_sized_cell_and_time(builder):
    """10,000-atom LiMnO2 cell (BASELINE configs[3]): identical to the host C++ builder, and the build time on the device."""
    z, frac, lat = graphgen.limno2_structure((10, 5, 25), 0.02, 4000)
    ag, img, d2u, u2d, bg = graphgen.native_graph_arrays(frac, lat, 6.0, 3.0)
    f64 = torch.as_tensor(frac).cuda().contiguous()
    out = builder.graph_arrays(f64, lat)
    assert builder.last_sizes == (len(ag), len(u2d), len(bg))
    assert np.array_equal(torch.stack([out["center"], out["nbr"]], 1).cpu().numpy(), ag)
    assert np.array_equal(out["image"].cpu().numpy(), img) and np.array_equal(out["d2u"].cpu().numpy(), d2u)
    assert np.array_equal(out["u2d"].cpu().numpy(), u2d)
    got_bg = torch.stack([out[k] for k in ("ang_atom", "ang_i", "ang_di", "ang_j", "ang_dj")], 1).cpu().numpy()
    assert np.array_equal(got_bg, bg)
    for _ in range(3):
        builder.graph_arrays(f64, lat)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(10):
        builder.graph_arrays(f64, lat)
    e.record()
    e.synchronize()
    ms = s.elapsed_time(e) / 10
    print(f"device graph build, 10,000 atoms ({len(ag)} edges, {len(bg)} angles): {ms:.3f} ms per build")
    assert ms < 10.0


def test_model_gives_the_same_answer_through_the_device_builder(builder):
    import os

    from chgnet_b200.model import CHGNet

    gold = os.path.join(os.path.dirname(__file__), "golden", "chgnet_0.3.0_weights.npz")
    model = CHGNet.from_file(gold, version="0.3.0").to("cuda")
    z, frac, lat = graphgen.limno2_structure((3, 2, 2), 0.03, 4100)
    host = model.predict_graph(graphgen.make_crystal_graph(z, frac, lat), task="efsm")
    batch = builder.build_batch(z, torch.as_tensor(frac).cuda().contiguous(), lat)
    res = model._get_native()(batch, need_grad=True, need_magmom=True)
    torch.cuda.synchronize()
    e = float((res["energy"] + res["e_ref"])[0]) / len(z)
    assert abs(e - float(host["e"])) < 1e-5
    assert np.abs(res["force"].float().cpu().numpy() - host["f"]).max() < 1e-4
    assert np.abs(res["magmom"].cpu().numpy() - host["m"]).max() < 1e-4


def test_predict_structure_device_and_host_graph_paths_agree(monkeypatch):
    """CHGNet.predict_structure builds the graph on the device by default; CHGNET_B200_GRAPH=host selects the host
    converter.  Same graph bit for bit -> same numbers; isolated atoms raise like the reference's converter
    (converter.py:160-174)."""
    import os

    from chgnet_b200.model import CHGNet

    gold = os.path.join(os.path.dirname(__file__), "golden", "chgnet_0.3.0_weights.npz")
    model = CHGNet.from_file(gold, version="0.3.0").to("cuda")
    z, frac, lat = graphgen.random_structure(31, 9720)
    dev = model.predict_structure((z, frac, lat), task="efsm", return_site_energies=True, return_crystal_feas=True)
    monkeypatch.setenv("CHGNET_B200_GRAPH", "host")
    host = model.predict_structure((z, frac, lat), task="efsm", return_site_energies=True, return_crystal_feas=True)
    monkeypatch.delenv("CHGNET_B200_GRAPH")
    assert set(dev) == set(host)
    for k in host:
        assert dev[k].shape == host[k].shape, k
        assert np.abs(np.asarray(dev[k], np.float64) - np.asarray(host[k], np.float64)).max() < 1e-5, k
    with pytest.raises(ValueError, match="isolated atom"):
        model.predict_structure(([1, 1], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 20.0))
    with pytest.raises(IndexError, match="index out of range"):
        model.predict_structure(([3, 99], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 4.0))


def test_predict_structure_of_a_list_native_builder_equals_converter_loop(monkeypatch):
    """predict_structure(list) builds the graphs of a chunk concurrently in the library and packs them out of the
    builder's memory (CHGNet.structures_to_batch); CHGNET_B200_GRAPH=python converts structure by structure like the
    reference (model.py:578-583).  Same batches -> same numbers, per structure, in order; chunking by batch_size."""
    import os

    from chgnet_b200.model import CHGNet

    gold = os.path.join(os.path.dirname(__file__), "golden", "chgnet_0.3.0_weights.npz")
    model = CHGNet.from_file(gold, version="0.3.0").to("cuda")
    structs = [graphgen.random_structure(n, 9800 + n) for n in (7, 31, 18, 40, 12, 25, 9)]
    native = model.predict_structure(structs, task="efsm", return_site_energies=True, batch_size=3)
    monkeypatch.setenv("CHGNET_B200_GRAPH", "python")
    loop = model.predict_structure(structs, task="efsm", return_site_energies=True, batch_size=3)
    monkeypatch.delenv("CHGNET_B200_GRAPH")
    assert len(native) == len(loop) == len(structs)
    for a, b, s in zip(native, loop, structs):
        assert set(a) == set(b)
        assert a["f"].shape == (len(s[0]), 3)
        for k in b:
            assert a[k].shape == b[k].shape, k
            assert np.abs(np.asarray(a[k], np.float64) - np.asarray(b[k], np.float64)).max() < 1e-6, k
    with pytest.raises(ValueError, match="isolated atom"):
        model.predict_structure(structs[:2] + [([1, 1], np.array([[0.0, 0, 0], [0.5, 0.5, 0.5]]), np.eye(3) * 20.0)])
