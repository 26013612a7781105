"""-m gpu: every architecture variant of tests/arch_variants.py on the H100, against fp64.

* Kernel replay: every kernel call of an inference run, an e/m training step, an e/f/s/m training step (second-order
  pass) and a Hessian-vector run, recorded on the torch specifications and replayed through the CUDA library under the
  default dispatch with ``ws_min_rows`` 0 (the tensor-core message kernels run on these small batches too), each output
  checked against the fp64 evaluation of its specification (tests/replay_fp64.py, its R, K and OVERRIDES).  The
  largest basis and the 8-block model also replay one batch above 4096 edges and angles at the default options.
* End to end: ``predict_graph`` on the native path, on the Python schedule and through one ``static_evaluator`` call
  against the fp64 oracle fed the same state_dict.  The native workspace is filled with NaN before the compared calls,
  so a kernel that reads workspace nobody wrote fails instead of passing on zeroed memory.
* ``Trainer.train_step`` and ``predict_hessian`` for the variants that change what they differentiate."""
import numpy as np
import pytest
import torch

from arch_variants import VARIANTS, architecture, cells, cutoffs, new_model, trainable_names
from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights
from oracle import chgnet_oracle as orc

pytestmark = pytest.mark.gpu

# north-star tolerances (BASELINE.json), x5 for random weights as in test_model_gpu.py::test_v020_shaped_architecture_end_to_end
TOL = {"e": 1e-4, "f": 1e-3, "s": 1e-3, "m": 1e-3}
RANDOM_WEIGHTS = 5.0
GRAD_RTOL = 1e-2  # test_train_gpu.py::test_trainer_efsm_step_matches_reference_combined_loss
HESSIAN_TOL = 2e-3  # test_hessian_gpu.py::TOL


def _second_order_recorder():
    """RecordingKernels that also records the Hessian-vector and strain second-derivative kernels"""
    import replay_fp64
    from kernel_replay import RecordingKernels

    from oracle.elastic import ElasticSpecKernels

    class Recorder(RecordingKernels, ElasticSpecKernels):
        recorded = replay_fp64.ALL_OUT_ARGS

    return Recorder()


def _record_and_check(variant, runs, graphs, ws_min_rows=None):
    """Record ``runs`` of the Python schedule on ``graphs`` and replay + check each call as it is recorded."""
    import replay_fp64

    from chgnet_b200._lib import CudaKernels

    w, args, margs = architecture(variant)
    has_m = args["n_conv"] > 1
    K = CudaKernels()
    chk = replay_fp64.Checker()
    rec = _second_order_recorder()
    rec.calls = replay_fp64.StreamedCalls(K, chk)
    eng = Engine(pack_weights({k: torch.as_tensor(v) for k, v in w.items()}, margs, device="cpu"), rec)
    compact = not margs.get("mlp_out_bias", False)
    n, nb = sum(g.atomic_number.shape[0] for g in graphs), len(graphs)
    gen = torch.Generator().manual_seed(21)
    try:
        if ws_min_rows is not None:
            K.set_option("ws_min_rows", ws_min_rows)
        if "inference" in runs:
            eng.run(build_batch(graphs, "cpu", compact_bonds=compact), need_grad=True, need_magmom=has_m,
                    need_atom_fea=has_m, need_crystal_fea=True)
        if "train" in runs:
            cm = (lambda: torch.randn(n, generator=gen)) if has_m else (lambda: None)
            out = eng.run(build_batch(graphs, "cpu", compact_bonds=compact), need_grad=True, need_magmom=has_m, train=True)
            eng.param_grads(out, torch.randn(nb, generator=gen), cm())
            out = eng.run(build_batch(graphs, "cpu", compact_bonds=compact), need_grad=True, need_magmom=has_m, train=True)
            eng.input_grads(out, record=True)
            eng.param_grads(out, torch.randn(nb, generator=gen), cm(), torch.randn(n, 3, generator=gen),
                            torch.randn(nb, 3, 3, generator=gen))
        if "hvp" in runs:
            eng.hessian_vector_products(build_batch(graphs, "cpu", compact_bonds=compact), torch.randn(n, 3, generator=gen))
    finally:
        K.set_option("ws_min_rows", 4096)
    title = f"{variant} ({', '.join(runs)}{'' if ws_min_rows is None else f', ws_min_rows={ws_min_rows}'})"
    chk.assert_ok(title)
    worst = max(((v[1], k) for k, v in chk.worst.items()), default=(0.0, None))
    print(f"{title}: worst err/tol {worst[0]:.3f} at {worst[1]}")
    return chk


@pytest.mark.parametrize("variant", VARIANTS)
def test_kernel_replay_matches_fp64(variant):
    from kernel_replay import SECOND_ORDER_KERNELS

    chk = _record_and_check(variant, ("inference", "train", "hvp"), cells(variant, seed=9600, n_lo=8, n_hi=16), ws_min_rows=0)
    want = {"atom_conv_fused", "readout", "force_virial", "readout_bwd", "wgrad", "bond_basis_hvp", "edge_tangent_bwd",
            "angle_basis_embed"} | SECOND_ORDER_KERNELS
    n_conv = VARIANTS[variant].get("n_conv", 4)
    if n_conv == 1:  # no BondConv, no angle adjoint
        want -= {"bond_conv_tan", "bond_conv_bwd2", "angle_basis_bwd2"}
        assert not {"bond_conv_fused", "angle_basis_bwd", "angle_basis_hvp"} & chk.kernels, sorted(chk.kernels)
    else:
        want |= {"bond_conv_fused", "angle_basis_bwd", "angle_basis_hvp"}
    if n_conv <= 2:  # the one AngleUpdate of two blocks is the dead last one
        want -= {"angle_update_tan", "angle_update_bwd2"}
        assert not {"angle_update_fwd", "angle_update_bwd"} & chk.kernels, sorted(chk.kernels)
    else:
        want |= {"angle_update_fwd", "angle_update_bwd"}
    if VARIANTS[variant].get("num_angular") == 1:  # the only output of angle_basis_bwd2, g_freq, has no entries
        want -= {"angle_basis_bwd2"}
    assert want <= chk.kernels, sorted(want - chk.kernels)


@pytest.mark.parametrize("variant", ["basis-32-31", "conv-8"])
def test_kernel_replay_above_4096_rows_matches_fp64(variant):
    """144-atom LiMnO2 (3x3x2, rattled) and a random cell: above 4096 edges and angles, so the default dispatch takes
    the tensor-core kernels by itself"""
    z, frac, lat = graphgen.limno2_structure((3, 3, 2), 0.02, 5)
    cut = cutoffs(variant)
    graphs = [graphgen.make_crystal_graph(z, frac, lat, **cut)] + graphgen.random_graphs(1, 20, 20, 9650, **cut)
    b = build_batch(graphs, "cpu")
    assert b.n_edges > 4096 and b.n_angles > 4096, (b.n_edges, b.n_angles)
    _record_and_check(variant, ("inference",), graphs)


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def _worst(preds, ref, graphs, is_intensive):
    out = {}
    for k in TOL:
        errs = []
        for p, r, g in zip(preds, ref, graphs):
            if k not in r:
                continue
            d = np.abs(np.asarray(p[k], dtype=np.float64) - np.asarray(r[k], dtype=np.float64))
            if k == "e" and not is_intensive:
                d = d / len(g.atomic_number)  # the tolerance is per atom
            errs.append(float(d.max()) if d.size else 0.0)
        if errs:
            out[k] = max(errs)
    return out


@pytest.fixture(scope="module", params=list(VARIANTS))
def end_to_end(request):
    """(variant, model on the GPU, graphs, task, fp64 oracle predictions)"""
    variant = request.param
    w, args, _ = architecture(variant)
    task = "efsm" if args["n_conv"] > 1 else "efs"
    graphs = cells(variant, seed=9700, n=4, n_lo=8, n_hi=20)
    ref = orc.predict_graph(w, graphs, task, batch_size=len(graphs), dtype=torch.float64, args=args, device="cuda")
    return variant, new_model(variant, "cuda"), graphs, task, ref


def _assert_close(label, preds, ref, graphs, variant):
    worst = _worst(preds, ref, graphs, architecture(variant)[1]["is_intensive"])
    print(f"{variant} {label}: max |cuda - oracle64| =", {k: f"{v:.2e}" for k, v in worst.items()})
    for k, v in worst.items():
        assert v < TOL[k] * RANDOM_WEIGHTS, (variant, label, k, v)
    assert set(worst) == set(ref[0]) & set(TOL)


def test_native_predict_graph_matches_oracle(end_to_end):
    variant, model, graphs, task, ref = end_to_end
    model.predict_graph(graphs, task=task, batch_size=len(graphs))  # sizes the workspace
    nat = model._get_native()
    calls = nat.calls
    nat.workspace.fill_(0xFF)  # NaN everywhere: reading stale workspace cannot pass by luck
    preds = model.predict_graph(graphs, task=task, batch_size=len(graphs))
    assert nat.calls == calls + 1
    _assert_close("native", preds, ref, graphs, variant)


def test_python_schedule_matches_oracle(end_to_end, monkeypatch):
    variant, model, graphs, task, ref = end_to_end
    monkeypatch.setenv("CHGNET_B200_ENGINE", "python")
    calls = model._get_native().calls
    preds = model.predict_graph(graphs, task=task, batch_size=len(graphs))
    assert model._get_native().calls == calls  # the Python schedule really ran
    _assert_close("python schedule", preds, ref, graphs, variant)


def test_static_evaluator_matches_oracle(end_to_end):
    variant, model, graphs, task, ref = end_to_end
    ev = model.static_evaluator(graphs, task=task)
    ev()  # sizes the workspace (eager)
    model._get_native().workspace.fill_(0xFF)
    _assert_close("static_evaluator", ev(), ref, graphs, variant)


# ---------------------------------------------------------------------------------------------------------------------
# training step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["extensive", "frozen-rbf", "conv-1", "readout-4"])
def test_trainer_efsm_step_matches_oracle_autograd(variant):
    from chgnet_b200.trainer import Trainer

    w, args, _ = architecture(variant)
    has_m = args["n_conv"] > 1
    targets = "efsm" if has_m else "efs"
    model = new_model(variant, "cuda")
    graphs = graphgen.random_graphs(4, 8, 16, 9800, **cutoffs(variant))
    base = model.predict_graph(graphs, task=targets, batch_size=len(graphs))
    gen = torch.Generator().manual_seed(8)
    noisy = lambda v, a: torch.as_tensor(np.asarray(v), dtype=torch.float32) + a * torch.randn(np.asarray(v).shape, generator=gen)  # noqa: E731
    lab = {"e": noisy([float(p["e"]) for p in base], 0.05), "f": [noisy(p["f"], 0.02) for p in base],
           "s": [noisy(p["s"], 0.05) for p in base]}
    if has_m:
        lab["m"] = [noisy(p["m"], 0.05) for p in base]
    trainable = trainable_names(variant)
    P = {k: torch.as_tensor(v).double().requires_grad_(k in trainable) for k, v in w.items()}
    o = orc.forward(P, graphs, targets, dtype=torch.float64, train=True, args=args)
    mse = torch.nn.MSELoss()
    loss = (mse(lab["e"].double(), o["e"]) + mse(torch.cat(lab["f"]).double(), torch.cat(o["f"]))
            + 0.1 * mse(torch.stack(lab["s"]).double(), torch.stack(o["s"])))
    if has_m:
        loss = loss + 0.1 * mse(torch.cat(lab["m"]).double(), torch.cat(o["m"]))
    names = sorted(trainable)
    want = dict(zip(names, torch.autograd.grad(loss, [P[k] for k in names], allow_unused=True)))

    trainer = Trainer(model, targets=targets, criterion="MSE", learning_rate=1e-5)
    assert sorted(trainer.names) == names
    frozen = {n: b.clone() for n, b in model.named_buffers()}
    report = trainer.train_step(graphs, lab)
    assert report["loss"] == pytest.approx(float(loss.detach()), rel=5e-3, abs=1e-7)
    got = trainer.grads_by_name()
    worst = 0.0
    for k in names:
        wk = want[k] if want[k] is not None else torch.zeros_like(P[k])
        if wk.numel() == 0:
            continue
        scale = float(wk.abs().max())
        err = float((got[k].double().cpu() - wk).abs().max())
        worst = max(worst, err / scale if scale > 0 else err)
        assert err <= GRAD_RTOL * scale + 1e-7, (k, err, scale)
    print(f"{variant}: train_step loss {report['loss']:.6f} (oracle {float(loss):.6f}), worst relative gradient error {worst:.2e}")
    for n, b in model.named_buffers():  # frozen basis frequencies stay as they are
        assert torch.equal(b, frozen[n]), n


# ---------------------------------------------------------------------------------------------------------------------
# Hessian
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["conv-1", "readout-1", "readout-4", "ln-gmlp-only", "ln-readout-only"])
def test_predict_hessian_matches_oracle(variant):
    from oracle.hessian import oracle_hessian

    w, args, _ = architecture(variant)
    model = new_model(variant, "cuda")
    z, frac, lat = graphgen.random_structure(8, 9900)
    g = graphgen.make_crystal_graph(z, frac, lat, **cutoffs(variant))
    assert len(g.bond_graph) > 0
    h = model.predict_hessian(g)
    want = oracle_hessian(w, g, args)
    scale = np.abs(want).max()
    n = len(z)
    fig = dict(err=np.abs(h - want).max() / scale, asym=np.abs(h - h.T).max() / scale,
               acoustic=np.abs(h.reshape(3 * n, n, 3).sum(axis=1)).max() / scale)
    print(variant, "Hessian", {k: f"{v:.2e}" for k, v in fig.items()})
    assert max(fig.values()) <= HESSIAN_TOL, fig
