"""-m gpu: Hessian-vector products and force constants on the device.

* every kernel call of a Hessian-vector run, replayed through the CUDA library against its torch specification;
* ``CHGNet.predict_hessian`` against the fp64 oracle's double-backward Hessian (LiMnO2 with its collinear bond
  pairs, a 31-atom random cell, and the 0.2.0 weights whose bond graph is not compacted);
* ``hessian_vector_product`` = the same columns of ``predict_hessian``; a rigid translation costs nothing;
  ``CHGNetCalculator.get_hessian`` = ``predict_hessian``."""
import json
import os

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights
from oracle import chgnet_oracle as orc
from oracle.hessian import oracle_hessian

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
# max error, asymmetry and acoustic-sum residual of the fp32 device Hessian, as fractions of max|H|
TOL = 2e-3
# positional indices of the output (accumulated) arguments of the Hessian-vector kernels
HVP_OUT_ARGS = {"bond_basis_hvp": [12], "angle_basis_hvp": [7], "edge_tangent_bwd": [10]}


def _recording_kernels():
    from kernel_replay import OUT_ARGS, RecordingKernels

    from oracle.hessian import HessianSpecKernels

    class HvpRecordingKernels(RecordingKernels, HessianSpecKernels):
        recorded = {**OUT_ARGS, **HVP_OUT_ARGS}

    return HvpRecordingKernels()


def test_every_hvp_kernel_matches_its_spec(weights030):
    import replay_fp64
    from kernel_replay import OUT_ARGS

    from chgnet_b200._lib import CudaKernels

    graphs = graphgen.random_graphs(3, 10, 16, 9700)
    n = sum(g.atomic_number.shape[0] for g in graphs)
    rec = _recording_kernels()
    eng = Engine(pack_weights({k: torch.as_tensor(v) for k, v in weights030.items()}, None, device="cpu"), rec)
    v = torch.randn(n, 3, generator=torch.Generator().manual_seed(5))
    eng.hessian_vector_products(build_batch(graphs, "cpu"), v)
    chk = replay_fp64.Checker()
    replay_fp64.replay(rec.calls, CudaKernels(), chk)
    chk.assert_ok("Hessian-vector products")
    assert set(HVP_OUT_ARGS) <= chk.kernels and chk.kernels <= set(OUT_ARGS) | set(HVP_OUT_ARGS), sorted(chk.kernels)


def _figures(h, want):
    scale = np.abs(want).max()
    n = h.shape[0] // 3
    return dict(err=np.abs(h - want).max() / scale, asym=np.abs(h - h.T).max() / scale,
                acoustic=np.abs(h.reshape(3 * n, n, 3).sum(axis=1)).max() / scale)


@pytest.fixture(scope="module")
def model030():
    from chgnet_b200.model import CHGNet

    return CHGNet.from_file(os.path.join(GOLD, "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")


@pytest.mark.parametrize("cell", ["limno2", "random31"])
def test_predict_hessian_matches_oracle(model030, weights030, cell):
    if cell == "limno2":
        z, frac, lat = graphgen.limno2_structure()
    else:
        z, frac, lat = graphgen.random_structure(31, 9731)
    g = graphgen.make_crystal_graph(z, frac, lat)
    h = model030.predict_hessian(g)
    assert h.shape == (3 * len(z), 3 * len(z)) and h.dtype == np.float64
    fig = _figures(h, oracle_hessian(weights030, g))
    print(cell, {k: f"{v:.2e}" for k, v in fig.items()})
    assert max(fig.values()) <= TOL, fig
    # structure input: the graph is built by the model's converter; a batch_size that does not divide 3N
    h2 = model030.predict_hessian((z, frac, lat), batch_size=5)
    assert np.abs(h2 - h).max() <= 1e-4 * np.abs(h).max()


def test_predict_hessian_020_uncompacted_bonds():
    from chgnet_b200.model import CHGNet

    w = orc.load_weights_npz(os.path.join(GOLD, "chgnet_0.2.0_weights.npz"))
    margs = json.loads(str(w["__model_args__"]))
    keys = ("num_radial", "num_angular", "gMLP_norm", "readout_norm", "mlp_out_bias", "cutoff_coeff",
            "atom_graph_cutoff", "bond_graph_cutoff", "n_conv", "is_intensive")
    args = {k: margs[k] for k in keys if k in margs}
    model = CHGNet.from_file(os.path.join(GOLD, "chgnet_0.2.0_weights.npz")).to("cuda")
    assert model._arch.get("mlp_out_bias", False)  # every bond carries a BondConv update: no compaction
    z, frac, lat = graphgen.limno2_structure()
    g = graphgen.make_crystal_graph(z, frac, lat, atom_graph_cutoff=float(margs["atom_graph_cutoff"]),
                                    bond_graph_cutoff=float(margs["bond_graph_cutoff"]))
    fig = _figures(model.predict_hessian(g), oracle_hessian(w, g, args))
    print("0.2.0", {k: f"{v:.2e}" for k, v in fig.items()})
    assert max(fig.values()) <= TOL, fig


def test_hvp_columns_translation_and_calculator(model030):
    from chgnet_b200.dynamics import Atoms, CHGNetCalculator

    z, frac, lat = graphgen.limno2_structure()
    g = graphgen.make_crystal_graph(z, frac, lat)
    n = len(z)
    h = model030.predict_hessian(g)
    scale = np.abs(h).max()
    cols = [0, 5, 13, 3 * n - 1]
    v = np.zeros((len(cols), n, 3))
    for k, c in enumerate(cols):
        v.reshape(len(cols), -1)[k, c] = 1.0
    hv = model030.hessian_vector_product(g, v)
    assert hv.shape == v.shape and hv.dtype == np.float64
    assert np.abs(hv.reshape(len(cols), -1).T - h[:, cols]).max() <= TOL * scale
    one = model030.hessian_vector_product(g, v[1])
    assert one.shape == (n, 3) and np.abs(one - hv[1]).max() <= TOL * scale
    shift = np.tile(np.array([0.3, -0.5, 0.8]), (n, 1))  # a rigid translation: every edge tangent is zero
    assert np.abs(model030.hessian_vector_product(g, shift)).max() <= TOL * scale
    calc = CHGNetCalculator(model=model030)
    atoms = Atoms(z, frac @ lat, lat)
    assert np.abs(calc.get_hessian(atoms) - model030.predict_hessian((z, frac, lat))).max() <= 1e-4 * scale
    with pytest.raises(ValueError):
        model030.hessian_vector_product(g, np.zeros((n + 1, 3)))
