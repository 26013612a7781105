"""The fp64 replay rule (tests/replay_fp64.py) has teeth: small errors planted in the torch specification, whose fp32
outputs then stand in for a kernel's, are caught on every kernel output they change by more than 1e-4 of its scale,
and the unchanged fp32 specification passes."""
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights
from oracle import kernel_specs
from oracle.elastic import ElasticSpecKernels


@pytest.fixture(scope="module")
def recorded(weights030):
    """Every kernel call of a training step with energy and magmom seeds, then of one with force and stress seeds
    too, with its fp64 reference."""
    import replay_fp64
    from kernel_replay import RecordingKernels

    graphs = graphgen.random_graphs(2, 8, 12, 9500)
    rec = RecordingKernels()
    eng = Engine(pack_weights({k: torch.as_tensor(v) for k, v in weights030.items()}, None, device="cpu"), rec)
    gen = torch.Generator().manual_seed(11)
    n_atoms = sum(g.atomic_number.shape[0] for g in graphs)
    out = eng.run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True, train=True)
    eng.param_grads(out, torch.randn(len(graphs), generator=gen), torch.randn(n_atoms, generator=gen))
    out = eng.run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True, train=True)
    eng.input_grads(out, record=True)
    eng.param_grads(out, torch.randn(len(graphs), generator=gen), torch.randn(n_atoms, generator=gen),
                    torch.randn(n_atoms, 3, generator=gen), torch.randn(len(graphs), 3, 3, generator=gen))
    return [(name, snap, outs, replay_fp64.reference64(name, snap)) for name, snap, outs in rec.calls]


def _spec32(name, snap):
    args = [a.clone() if isinstance(a, torch.Tensor) else a for a in snap]
    getattr(ElasticSpecKernels(), name)(*args)
    return args


def _scaled(fn, factor):
    return lambda *a: fn(*a) * factor


MUTATIONS = {
    "ln_bwd*(1+1e-3)": ("_ln_bwd", lambda f: _scaled(f, 1 + 1e-3)),
    "gate_bwd*(1+1e-2)": ("_gate_bwd", lambda f: _scaled(f, 1 + 1e-2)),
    "d2silu=0": ("_d2silu", lambda f: (lambda x: torch.zeros_like(x))),
    "dsig*(1+1e-3)": ("_dsig", lambda f: _scaled(f, 1 + 1e-3)),
}


def test_unchanged_fp32_spec_passes(recorded):
    import replay_fp64

    chk = replay_fp64.Checker()
    for name, snap, outs, ref in recorded:
        chk.check_call(name, _spec32(name, snap), ref, outs)
    chk.assert_ok("unchanged fp32 specification")
    from kernel_replay import TRAIN_KERNELS

    assert TRAIN_KERNELS <= chk.kernels


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_planted_error_is_caught(recorded, mutation, monkeypatch):
    import replay_fp64

    attr, make = MUTATIONS[mutation]
    monkeypatch.setattr(kernel_specs, attr, make(getattr(kernel_specs, attr)))
    chk = replay_fp64.Checker()
    changed, missed = set(), []
    for name, snap, outs, ref in recorded:
        args = _spec32(name, snap)
        for idx, want in ref.items():
            scale = float(want.abs().max()) if want.numel() else 0.0
            delta = float((args[idx].double() - outs[idx].double()).abs().max()) if want.numel() else 0.0
            flagged = not chk.check(name, idx, args[idx], want, outs[idx])
            if delta > 1e-4 * scale:
                changed.add((name, idx))
                if not flagged:
                    missed.append(f"{name} out[{idx}]: changed by {delta / scale:.1e} of scale, not flagged")
    print(mutation, "caught on", sorted(changed))
    assert changed, f"{mutation} changed no output by more than 1e-4 of its scale"
    assert not missed, "\n".join(missed)
