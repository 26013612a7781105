"""CPU: every architecture the ``CHGNet`` constructor accepts, one variant per option, against the fp64 oracle.

The kernel checks elsewhere run the 0.3.0 shape (31 / 31 basis functions, 4 blocks, 3 readout layers, LayerNorm
everywhere, p = 8) and the 0.2.0 shape.  Here each variant changes one option of the 0.3.0 shape: basis sizes at the
lane limits (1 and 32 radial functions), 1 to 8 blocks, 1 to 4 readout layers, LayerNorm in the GatedMLPs only or in
the readout only, other envelope exponents and cutoffs, extensive energies and frozen basis frequencies
(tests/arch_variants.py).  Weights come from a seeded ``CHGNet(**variant).state_dict()``, re-drawn at the oracle's
random-weight scale; the cells are random cells built with the variant's cutoffs plus a dimer (edges, no angles) and an
isolated atom.

For each variant: the Python schedule on the torch kernel specifications in fp64 against the oracle (forward, forces,
stress, magmoms, features), the native host packing and ``chg_forward_plan`` against the Python packing and call list,
and the parameter gradients of an e/m and an e/f/s/m loss against oracle autograd.  Shapes the kernels cannot run are
rejected when the model is built and when weights are packed."""
import numpy as np
import pytest
import torch

from arch_variants import VARIANTS, architecture, cells, fp64_batch, trainable_names
from chgnet_b200 import native
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import EV_A3_TO_GPA, Engine
from chgnet_b200.weights import pack_weights, unpack_grads
from oracle import chgnet_oracle as orc
from oracle.kernel_specs import SpecKernels

TOL = 1e-9  # test_engine_spec.py, fp64


def spec_engine(w, margs):
    sd = {k: torch.as_tensor(v).double() for k, v in w.items()}
    return Engine(pack_weights(sd, margs, device="cpu", dtype=torch.float64), SpecKernels()), sd


# ---------------------------------------------------------------------------------------------------------------------
# forward + force / stress reverse pass
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
def test_forward_matches_oracle_fp64(variant):
    w, args, margs = architecture(variant)
    graphs = cells(variant)
    has_m = args["n_conv"] > 1  # magmoms are read after block n_conv - 1
    eng, _ = spec_engine(w, margs)
    b = fp64_batch(graphs)
    out = eng.run(b, need_grad=True, need_magmom=has_m, need_atom_fea=True, need_crystal_fea=True, keep_intermediates=True)
    ref = orc.forward(w, graphs, "efsm" if has_m else "efs", dtype=torch.float64, args=args, return_atom_feas=True,
                      return_crystal_feas=True, return_intermediates=True)
    n = torch.tensor(b.atoms_per_graph, dtype=torch.float64)
    # AtomRef is evaluated in fp32 by the reference even for an fp64 model (composition_model.py:191): the same
    # per-atom tolerance as test_engine_spec.py, summed over the atoms of an extensive energy
    if args["is_intensive"]:
        assert torch.allclose((out.energy + out.e_ref) / n, ref["e"].double(), atol=2e-6, rtol=0)
    else:
        assert bool(((out.energy + out.e_ref - ref["e"].double()).abs() <= 2e-6 * n).all())
    e_model = torch.zeros(len(graphs), dtype=torch.float64).index_add_(0, b.owner.long(), ref["intermediates"]["site_e_model"])
    assert torch.allclose(out.energy, e_model, atol=TOL * 100, rtol=0), (out.energy - e_model).abs().max()
    f_ref = torch.cat(ref["f"])
    assert torch.allclose(out.force, f_ref, atol=TOL * 10, rtol=0), (out.force - f_ref).abs().max()
    assert float(f_ref.abs().max()) > 1e-3  # the forces are not trivially zero
    s = out.virial.view(-1, 3, 3) * (EV_A3_TO_GPA / b.volume)[:, None, None]
    assert torch.allclose(s, torch.stack(ref["s"]), atol=TOL * 100, rtol=0), (s - torch.stack(ref["s"])).abs().max()
    if has_m:
        assert torch.allclose(out.magmom, torch.cat(ref["m"]), atol=TOL * 10)
        assert torch.allclose(out.atom_fea, torch.cat(ref["atom_fea"]), atol=TOL * 10)
    else:
        assert out.magmom is None and out.atom_fea is None and "m" not in ref and "atom_fea" not in ref
    assert torch.allclose(out.crystal_fea, ref["crystal_fea"], atol=TOL * 100)
    compared = 0
    for k, v in ref["intermediates"].items():
        if v is not None and out.extras.get(k) is not None:
            assert torch.allclose(out.extras[k], v, atol=TOL * 10, rtol=TOL * 10), k
            compared += 1
    assert compared >= 3 * args["n_conv"] + 2, compared


# ---------------------------------------------------------------------------------------------------------------------
# native host packing and schedule
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
def test_native_packing_matches_python_packing(variant):
    w, args, margs = architecture(variant)
    sd = {k: torch.as_tensor(v) for k, v in w.items()}
    pw = pack_weights(sd, margs, device="cpu")
    hps, blob, hp = native.pack_weights_native(sd, margs)
    lay = native.packed_layout(hps)
    assert lay["__total__"][0] == blob.numel()
    hidden = VARIANTS[variant].get("mlp_hidden_dims", (64, 64, 64))
    assert (hps.num_radial, hps.num_angular, hps.n_conv, hps.cutoff_coeff, hps.n_readout_hidden) == (
        args["num_radial"], args["num_angular"], args["n_conv"], args["cutoff_coeff"], len(np.atleast_1d(hidden)))
    assert (bool(hps.use_ln), bool(hps.readout_ln)) == (args["gMLP_norm"] == "layer", args["readout_norm"] == "layer")
    assert (hps.atom_graph_cutoff, hps.bond_graph_cutoff) == pytest.approx((args["atom_graph_cutoff"], args["bond_graph_cutoff"]))
    assert hp.is_intensive == args["is_intensive"] and pw.mlp_wt.shape[0] == hps.n_readout_hidden

    def same(name, t):
        if t is None:
            assert name not in lay, name
            return
        off, n = lay[name]
        assert n == t.numel() and torch.equal(blob[off:off + n], t.reshape(-1).float()), name

    for name in ("emb", "freq_ag", "freq_bg", "freq_ang", "w3t", "w3", "wang_t", "wang", "readout_ln", "mlp_wt", "mlp_w",
                 "mlp_b", "w_last", "w_mag", "atom_ref"):
        same(name, getattr(pw, name))
    assert hps.b_last == pytest.approx(pw.b_last) and hps.b_mag == pytest.approx(pw.b_mag)
    assert (len(pw.atom), len(pw.bond), len(pw.angle)) == (args["n_conv"], args["n_conv"] - 1, args["n_conv"] - 1)
    for kind, packs in (("atom", pw.atom), ("bond", pw.bond), ("angle", pw.angle)):
        for t, gp in enumerate(packs):
            k = f"{kind}.{t}"
            if kind != "angle":
                same(f"{k}.w2t", gp.w2t), same(f"{k}.w2", gp.w2), same(f"{k}.b2", gp.b2)
                same(f"{k}.wo_t", gp.extra["wo_t"]), same(f"{k}.wo", gp.extra["wo"]), same(f"{k}.bo", gp.extra["bo"])
            same(f"{k}.ln", gp.ln)
            names = ("wcn_t", "we_t", "b1", "wcn_b", "we_b") if kind == "atom" else \
                ("wij_t", "bij", "wx_t", "w1a_t", "wij_b", "wx_b", "w1a_b")
            for name in names:
                same(f"{k}.{name}", gp.extra[name])


# the three flag sets of test_native_cpu.py
FLAGS = [dict(need_grad=True, need_magmom=True), dict(need_grad=False, need_crystal_fea=True, need_atom_fea=True),
         dict(need_grad=True)]


@pytest.mark.parametrize("variant", VARIANTS)
def test_native_plan_is_the_python_schedule(variant):
    from kernel_replay import RecordingKernels

    w, args, margs = architecture(variant)
    sd = {k: torch.as_tensor(v) for k, v in w.items()}
    hps, _, _ = native.pack_weights_native(sd, margs)
    graphs = cells(variant)
    g_iso = graphs[2]
    for flags in FLAGS:
        flags = dict(flags)
        if args["n_conv"] == 1:
            flags.pop("need_magmom", None)
        wanted = native.Outputs(energy=1, e_ref=1, site_e=1, magmom=1 if flags.get("need_magmom") else None,
                                atom_fea=1 if flags.get("need_atom_fea") else None,
                                crystal_fea=1 if flags.get("need_crystal_fea") else None,
                                force=1 if flags["need_grad"] else None, virial=1 if flags["need_grad"] else None)
        for batch in (graphs, [g_iso]):
            b = build_batch(batch, "cpu")
            rec = RecordingKernels()
            Engine(pack_weights(sd, margs, device="cpu"), rec).run(b, **flags)
            need, got = native.plan(hps, native.batch_struct(b), wanted, want_trace=True)
            assert got == [name for name, _, _ in rec.calls], (flags, len(batch))
            assert need > 0


# ---------------------------------------------------------------------------------------------------------------------
# training gradients
# ---------------------------------------------------------------------------------------------------------------------
def _labels(graphs, ref, gen, has_m):
    """targets = the oracle's prediction + noise, in the reference's label layout flattened"""
    lab = {"e": ref["e"].detach() + 0.1 * torch.randn(len(graphs), generator=gen, dtype=torch.float64),
           "f": torch.cat(ref["f"]).detach() + 0.05 * torch.randn(sum(len(f) for f in ref["f"]), 3, generator=gen,
                                                                  dtype=torch.float64),
           "s": torch.stack(ref["s"]).detach() + 0.5 * torch.randn(len(graphs), 3, 3, generator=gen, dtype=torch.float64)}
    if has_m:
        lab["m"] = torch.cat(ref["m"]).detach() + 0.05 * torch.randn(len(lab["f"]), generator=gen, dtype=torch.float64)
    return lab


@pytest.mark.parametrize("targets", ["em", "efsm"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_param_grads_match_oracle_autograd(variant, targets):
    """CombinedLoss (MSE, the reference's ratios) through ``trainer.loss_and_grads`` on the spec engine in fp64 against
    autograd through the oracle; "efsm" takes the second-order pass.  The AtomRef is zeroed on both sides: the oracle
    rounds it to fp32 (composition_model.py:191), which would move the energy residual the gradients scale with."""
    from chgnet_b200.trainer import LossConfig, loss_and_grads

    w, args, margs = architecture(variant)
    w = dict(w, **{"composition_model.fc.weight": np.zeros((1, 94), dtype=np.float32)})
    has_m = args["n_conv"] > 1
    if not has_m:
        targets = targets.replace("m", "")
    graphs = cells(variant, seed=9400)
    trainable = trainable_names(variant)
    P = {k: torch.as_tensor(v).double().requires_grad_(k in trainable) for k, v in w.items()}
    out = orc.forward(P, graphs, "efsm" if has_m else "efs", dtype=torch.float64, train=True, args=args)
    lab = _labels(graphs, out, torch.Generator().manual_seed(11), has_m)
    mse = torch.nn.MSELoss()
    loss = mse(lab["e"], out["e"])
    if "m" in targets:
        loss = loss + 0.1 * mse(lab["m"], torch.cat(out["m"]))
    if "f" in targets:
        loss = loss + mse(lab["f"], torch.cat(out["f"])) + 0.1 * mse(lab["s"], torch.stack(out["s"]))
    names = sorted(trainable)
    want = dict(zip(names, torch.autograd.grad(loss, [P[k] for k in names], allow_unused=True)))

    eng, sd = spec_engine(w, margs)
    report, G = loss_and_grads(eng, fp64_batch(graphs), LossConfig(targets, "MSE"), lab, args["is_intensive"], False)
    got = unpack_grads(G, sd)
    assert report["loss"] == pytest.approx(float(loss.detach()), rel=1e-9)
    # first order: 1e-9 of the tensor's scale (test_train_spec.py); the second-order pass: 1e-6, second derivatives
    # near collinear bond pairs amplify rounding (acos' up to 700)
    rtol = 1e-6 if "f" in targets else 1e-9
    nonzero = 0
    for k in names:
        wk = want[k] if want[k] is not None else torch.zeros_like(P[k])
        if wk.numel() == 0:  # num_angular=1: no Fourier frequencies
            continue
        scale = max(float(wk.abs().max()), 1.0)
        assert float((got[k] - wk).abs().max()) <= rtol * scale, (k, float((got[k] - wk).abs().max()), scale)
        nonzero += float(wk.abs().max()) > 0
    assert nonzero >= len(names) // 2
    if not VARIANTS[variant].get("learnable_rbf", True):
        assert not any(k.endswith("frequencies") for k in names)


def test_frozen_frequencies_get_no_trainer_slot_and_stay_unchanged(monkeypatch):
    """learnable_rbf=False: the basis frequencies are buffers; a Trainer step (spec kernels injected) leaves them as
    they are and moves the parameters."""
    from arch_variants import new_model
    from chgnet_b200.trainer import Trainer

    model = new_model("frozen-rbf")
    eng = Engine(pack_weights(model.state_dict(), model.model_args, device="cpu"), SpecKernels())
    monkeypatch.setattr(model, "_get_engine", lambda: eng)
    trainer = Trainer(model, targets="efsm", criterion="MSE", learning_rate=1e-3)
    assert not any(n.endswith("frequencies") for n in trainer.names)
    freqs = {n: b.clone() for n, b in model.named_buffers() if n.endswith("frequencies")}
    assert len(freqs) == 3
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    graphs = cells("frozen-rbf", seed=9500, n=2)
    lab = {"e": torch.zeros(len(graphs)), "f": [torch.zeros(len(g.atomic_number), 3) for g in graphs],
           "s": [torch.zeros(3, 3) for _ in graphs], "m": [torch.zeros(len(g.atomic_number)) for g in graphs]}
    report = trainer.train_step(graphs, lab)
    assert np.isfinite(report["loss"])
    for n, b in model.named_buffers():
        if n in freqs:
            assert torch.equal(b, freqs[n]), n
    moved = {n for n, p in model.named_parameters() if p.requires_grad and not torch.equal(p.detach(), before[n])}
    # all but the last AngleUpdate, whose output is never read (model.py:470-496): zero gradient, no Adam step
    assert moved == {n for n in trainer.names if not n.startswith("angle_layers.2.")}


# ---------------------------------------------------------------------------------------------------------------------
# rejections
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw,exc,match", [
    (dict(num_radial=0), ValueError, "num_radial"),
    (dict(num_radial=40), ValueError, "num_radial"),
    (dict(num_angular=33), ValueError, "num_angular"),
    (dict(n_conv=0), ValueError, "n_conv"),
    (dict(n_conv=9), ValueError, "n_conv"),
    (dict(mlp_hidden_dims=(128, 64)), NotImplementedError, "mlp_hidden_dims"),
    (dict(mlp_hidden_dims=(32,)), NotImplementedError, "mlp_hidden_dims"),
    (dict(mlp_hidden_dims=[64] * 5), NotImplementedError, "mlp_hidden_dims"),
    (dict(mlp_hidden_dims=()), NotImplementedError, "mlp_hidden_dims"),
], ids=["num_radial-0", "num_radial-40", "num_angular-33", "n_conv-0", "n_conv-9", "readout-128-64", "readout-32",
        "readout-5-layers", "readout-0-layers"])
def test_constructor_rejects_shapes_the_kernels_cannot_run(kw, exc, match):
    from chgnet_b200.model import CHGNet

    with pytest.raises(exc, match=match):
        CHGNet(**kw)


def _with_readout(w: dict, widths) -> dict:
    """random oracle weights with the readout MLP replaced by hidden layers of ``widths`` (reference MLP layout)"""
    w = {k: v for k, v in w.items() if not k.startswith("mlp.layers.")}
    rng = np.random.default_rng(0)
    d = 64
    for i, h in enumerate(widths):
        w[f"mlp.layers.{2 * i}.weight"] = rng.standard_normal((h, d)).astype(np.float32) / np.sqrt(d)
        w[f"mlp.layers.{2 * i}.bias"] = np.zeros(h, np.float32)
        d = h
    w[f"mlp.layers.{2 * len(widths) + 1}.weight"] = rng.standard_normal((1, d)).astype(np.float32)
    w[f"mlp.layers.{2 * len(widths) + 1}.bias"] = np.zeros(1, np.float32)
    return w


@pytest.mark.parametrize("case,match", [
    ("readout-128-64", "mlp_hidden_dims"), ("readout-5-layers", "mlp_hidden_dims"), ("readout-32", "mlp_hidden_dims"),
    ("n_conv-9", "n_conv"), ("num_radial-40", "num_radial"), ("num_angular-33", "num_angular"),
])
def test_packing_rejects_weights_the_kernels_cannot_run(case, match):
    """state_dicts that reach the packers without the constructor (loaded weights): both the Python and the native
    packer refuse them, naming the argument, instead of reading a readout layer or a basis of the wrong shape"""
    base = orc.random_weights(1, dict(n_conv=2))
    w = {"readout-128-64": lambda: _with_readout(base, (128, 64)), "readout-5-layers": lambda: _with_readout(base, [64] * 5),
         "readout-32": lambda: _with_readout(base, (32,)), "n_conv-9": lambda: orc.random_weights(1, dict(n_conv=9)),
         "num_radial-40": lambda: orc.random_weights(1, dict(num_radial=40, n_conv=2)),
         "num_angular-33": lambda: orc.random_weights(1, dict(num_angular=33, n_conv=2))}[case]()
    sd = {k: torch.as_tensor(v) for k, v in w.items()}
    with pytest.raises((ValueError, NotImplementedError), match=match):
        pack_weights(sd, None, device="cpu")
    with pytest.raises((ValueError, NotImplementedError), match=match):
        native.pack_weights_native(sd, None)


def test_readout_depth_comes_from_the_layer_indices():
    """A hidden layer that is not 64 wide is not skipped: before this check (128, 64) was packed as ONE layer"""
    from chgnet_b200.weights import readout_layer_indices

    base = orc.random_weights(1, dict(n_conv=2))
    assert readout_layer_indices(base) == ([0, 2, 4], 7)
    assert readout_layer_indices(_with_readout(base, (128, 64))) == ([0, 2], 5)
    assert readout_layer_indices(_with_readout(base, [64])) == ([0], 3)


def test_one_block_model_refuses_magmoms():
    """n_conv=1: the reference reads magmoms after block n_conv - 1 (model.py:477-487), which one block does not have"""
    from chgnet_b200.model import CHGNet
    from chgnet_b200.trainer import Trainer

    model = CHGNet(n_conv=1)
    g = cells("conv-1")[0]
    for task in ("em", "efsm"):
        with pytest.raises(ValueError, match="n_conv"):
            model.predict_graph(g, task=task)
    with pytest.raises(ValueError, match="n_conv"):
        model([g], task="efsm")
    for targets in ("em", "efsm"):
        with pytest.raises(ValueError, match="n_conv"):
            Trainer(model, targets=targets)
    with pytest.raises(RuntimeError, match="no CPU path"):  # other tasks get as far as the device check
        model.predict_graph(g, task="efs")
