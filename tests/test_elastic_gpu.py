"""-m gpu: strain second derivatives and elastic tensors on the device.

* every kernel call of an ``Engine.second_derivatives`` run (position and strain directions mixed in one batch),
  replayed through the CUDA library against its torch specification, ``edge_tangent_bwd_virial`` included;
* ``CHGNet.predict_elastic_tensor`` against the fp64 oracle (LiMnO2 with its unstable mode, a 31-atom random cell,
  and the 0.2.0 weights whose bond graph is not compacted);
* its ``hessian`` = ``predict_hessian``; ``relaxed_ions=False`` = the clamped part of the full run;
* units and sign: central differences of ``predict_structure`` stresses under +-1e-4 Voigt strains = ``clamped_ion``."""
import json
import os
import warnings

import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights
from oracle import chgnet_oracle as orc
from oracle.elastic import VOIGT_PAIRS, oracle_elastic, voigt_directions

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
# clamped-ion tensor, internal strain and the asymmetry of C, as fractions of their max (the Hessian's tolerance)
TOL = 2e-3
# relaxed-ion tensor, as a fraction of max|C_relaxed|
TOL_RELAXED = 1e-2
# positional indices of the output (accumulated) arguments of the second-derivative geometry kernels
SD_OUT_ARGS = {"bond_basis_hvp": [12], "angle_basis_hvp": [7], "edge_tangent_bwd_virial": [12, 13]}


def _recording_kernels():
    from kernel_replay import OUT_ARGS, RecordingKernels

    from oracle.elastic import ElasticSpecKernels

    class SdRecordingKernels(RecordingKernels, ElasticSpecKernels):
        recorded = {**OUT_ARGS, **SD_OUT_ARGS}

    return SdRecordingKernels()


def test_every_second_derivatives_kernel_matches_its_spec(weights030):
    import replay_fp64
    from kernel_replay import OUT_ARGS

    from chgnet_b200._lib import CudaKernels

    # the 256-edge blocks at the two graph boundaries span two graphs: the virial takes its per-edge atomic path there
    graphs = graphgen.random_graphs(3, 10, 16, 9701)
    sizes = [g.atomic_number.shape[0] for g in graphs]
    gen = torch.Generator().manual_seed(6)
    v = torch.randn(sum(sizes), 3, generator=gen)
    v[: sizes[0]] = 0.0
    w = torch.randn(len(graphs), 3, 3, generator=gen)
    w[1] = 0.0
    rec = _recording_kernels()
    eng = Engine(pack_weights({k: torch.as_tensor(t) for k, t in weights030.items()}, None, device="cpu"), rec)
    eng.second_derivatives(build_batch(graphs, "cpu"), v, w)
    chk = replay_fp64.Checker()
    replay_fp64.replay(rec.calls, CudaKernels(), chk)
    chk.assert_ok("second derivatives")
    assert set(SD_OUT_ARGS) <= chk.kernels and chk.kernels <= set(OUT_ARGS) | set(SD_OUT_ARGS), sorted(chk.kernels)
    assert "edge_tangent_bwd" not in chk.kernels


def _figures(got, want):
    c, c_want = got["clamped_ion"], want["clamped_ion"]
    s_c = np.abs(c_want).max()
    fig = dict(clamped=np.abs(c - c_want).max() / s_c, asym=np.abs(c - c.T).max() / s_c,
               internal_strain=np.abs(got["internal_strain"] - want["internal_strain"]).max()
               / np.abs(want["internal_strain"]).max())
    rel = np.abs(got["relaxed_ion"] - want["relaxed_ion"]).max() / np.abs(want["relaxed_ion"]).max()
    return fig, rel


def _reduced_spectrum(h):
    """Eigenvalues of the symmetrised Hessian off the rigid translations (for the conditioning of C_relaxed)."""
    n = h.shape[0] // 3
    q = np.linalg.qr(np.tile(np.eye(3), (n, 1)), mode="complete")[0][:, 3:]
    return np.linalg.eigvalsh(q.T @ (0.5 * (h + h.T)) @ q)


@pytest.fixture(scope="module")
def model030():
    from chgnet_b200.model import CHGNet

    return CHGNet.from_file(os.path.join(GOLD, "chgnet_0.3.0_weights.npz"), version="0.3.0").to("cuda")


def _predict(model, g):
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always", RuntimeWarning)
        got = model.predict_elastic_tensor(g)
    return got, [w for w in caught if issubclass(w.category, RuntimeWarning)]


@pytest.mark.parametrize("cell", ["limno2", "random31"])
def test_predict_elastic_tensor_matches_oracle(model030, weights030, cell):
    if cell == "limno2":
        z, frac, lat = graphgen.limno2_structure()
    else:
        z, frac, lat = graphgen.random_structure(31, 9731)
    g = graphgen.make_crystal_graph(z, frac, lat)
    n = len(z)
    got, caught = _predict(model030, g)
    assert got["clamped_ion"].shape == (6, 6) and got["internal_strain"].shape == (3 * n, 6)
    assert got["relaxed_ion"].shape == (6, 6) and got["hessian"].shape == (3 * n, 3 * n)
    assert all(got[k].dtype == np.float64 for k in ("clamped_ion", "internal_strain", "relaxed_ion", "hessian"))
    want = oracle_elastic(weights030, g)
    fig, rel = _figures(got, want)
    spec = _reduced_spectrum(want["hessian"])
    print(cell, {k: f"{v:.2e}" for k, v in fig.items()}, f"relaxed {rel:.2e}", "unstable", got["unstable_modes"],
          want["unstable_modes"], f"reduced H eigenvalues: min {spec.min():.3g}, min|.| {np.abs(spec).min():.3g}, "
          f"max {spec.max():.3g}")
    assert max(fig.values()) <= TOL, fig
    assert rel <= TOL_RELAXED, rel
    assert got["unstable_modes"] == want["unstable_modes"]
    assert len(caught) == (1 if got["unstable_modes"] else 0)
    if cell == "limno2":
        assert got["unstable_modes"] == 1 and "1 unstable mode" in str(caught[0].message)
        # the hessian key is predict_hessian's matrix; the clamped-only run is the clamped part of the full run
        h = model030.predict_hessian(g)
        assert np.abs(got["hessian"] - h).max() <= 1e-4 * np.abs(h).max()
        clamped = model030.predict_elastic_tensor((z, frac, lat), relaxed_ions=False, batch_size=5)
        assert set(clamped) == {"clamped_ion", "internal_strain"}
        assert np.abs(clamped["clamped_ion"] - got["clamped_ion"]).max() <= 1e-4 * np.abs(got["clamped_ion"]).max()


def test_predict_elastic_tensor_020_uncompacted_bonds():
    from chgnet_b200.model import CHGNet

    w = orc.load_weights_npz(os.path.join(GOLD, "chgnet_0.2.0_weights.npz"))
    margs = json.loads(str(w["__model_args__"]))
    keys = ("num_radial", "num_angular", "gMLP_norm", "readout_norm", "mlp_out_bias", "cutoff_coeff",
            "atom_graph_cutoff", "bond_graph_cutoff", "n_conv", "is_intensive")
    args = {k: margs[k] for k in keys if k in margs}
    model = CHGNet.from_file(os.path.join(GOLD, "chgnet_0.2.0_weights.npz")).to("cuda")
    assert model._arch.get("mlp_out_bias", False)
    z, frac, lat = graphgen.limno2_structure()
    g = graphgen.make_crystal_graph(z, frac, lat, atom_graph_cutoff=float(margs["atom_graph_cutoff"]),
                                    bond_graph_cutoff=float(margs["bond_graph_cutoff"]))
    got, _ = _predict(model, g)
    want = oracle_elastic(w, g, args)
    fig, rel = _figures(got, want)
    print("0.2.0", {k: f"{v:.2e}" for k, v in fig.items()}, f"relaxed {rel:.2e}", "unstable", got["unstable_modes"])
    assert max(fig.values()) <= TOL, fig
    assert rel <= TOL_RELAXED, rel
    assert got["unstable_modes"] == want["unstable_modes"]


def test_clamped_ion_matches_stress_finite_differences(model030):
    """C_ab ~ d sigma_b / d e_a: central differences of the predicted stress under +-1e-4 Voigt strains.  They agree
    to terms of order the residual stress (~0.3 GPa on this cell) plus the fp32 stress noise over the step.  The step
    is 1e-4, not 1e-3: the fp64 oracle's own central differences at 1e-3 miss its exact C11 by 8 GPa (truncation),
    at 1e-4 every entry by at most 0.4 GPa."""
    z, frac, lat = graphgen.limno2_structure()
    c = model030.predict_elastic_tensor((z, frac, lat), relaxed_ions=False)["clamped_ion"]
    h, w = 1e-4, voigt_directions()
    fd = np.empty((6, 6))
    for a in range(6):
        s = []
        for sgn in (1.0, -1.0):
            strained = np.asarray(lat, dtype=np.float64) @ (np.eye(3) + sgn * h * w[a])
            sig = np.asarray(model030.predict_structure((z, frac, strained), task="efs")["s"], dtype=np.float64)
            sig = 0.5 * (sig + sig.T)
            s.append(np.array([sig[i, j] for i, j in VOIGT_PAIRS]))
        fd[a] = (s[0] - s[1]) / (2 * h)
    err = np.abs(fd - c).max()
    print("FD stress vs clamped_ion: max |diff| GPa", f"{err:.3f}", "max|C|", f"{np.abs(c).max():.1f}")
    assert err <= 3.0, (err, fd, c)
