"""The fp64 replay rule (tests/replay_fp64.py) has teeth: small errors planted in the torch specification, whose fp32
outputs then stand in for a kernel's, are caught on every kernel output they change by more than 1e-4 of its scale,
and the unchanged fp32 specification passes.  The guarded replay itself, run on the CPU through the fp32
specifications, flags each planted out-of-bounds or aliasing bug and passes the unplanted specifications."""
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


class FakeKernels(ElasticSpecKernels):
    """The fp32 specifications standing in for the CUDA library in ``replay_fp64.replay``, with at most one planted
    bug of the kind a kernel's index arithmetic gets wrong.  None of these changes a declared output element except
    the last, and that one only when the residual is ``y`` itself."""

    def __init__(self, bug: str | None = None) -> None:
        self.bug = bug

    def segment_sum(self, data, perm, ptr, accumulate, out):
        super().segment_sum(data, perm, ptr, accumulate, out)
        width = out.shape[1]
        if self.bug == "segment_sum writes width + 4 columns" and out.stride(0) > width:
            out.as_strided((out.shape[0], width + 4), out.stride())[:, width:] = 1.0

    def linear(self, x, wt, bias, residual, y, x_rows=None, y_rows=None):
        if self.bug == "linear adds the residual after storing y" and residual is not None:
            super().linear(x, wt, bias, None, y, x_rows, y_rows)
            rows = slice(None) if y_rows is None else y_rows.long()
            y[rows] += residual[rows]  # right for a separate residual; reads y back when the residual is y
            return
        super().linear(x, wt, bias, residual, y, x_rows, y_rows)
        if self.bug == "linear writes one row past the end of y":
            y.as_strided((y.shape[0] + 1, y.shape[1]), y.stride())[-1] = 1.0

    def wgrad(self, x, g, out, colsum=None, x_rows=None, g_rows=None, x_silu=False, x2=None):
        super().wgrad(x, g, out, colsum, x_rows, g_rows, x_silu, x2)
        if self.bug == "wgrad writes 128 columns" and out.stride(0) > out.shape[1]:
            out.as_strided((out.shape[0], 128), out.stride())[:, out.shape[1]:] = 1.0

    def atom_conv_fwd(self, pcn, pe, *args):
        super().atom_conv_fwd(pcn, pe, *args)
        if self.bug == "atom_conv_fwd zeroes pe after reading it":
            pe.zero_()


PLANTED = ["segment_sum writes width + 4 columns", "linear writes one row past the end of y",
           "wgrad writes 128 columns", "atom_conv_fwd zeroes pe after reading it",
           "linear adds the residual after storing y"]


def _replay_fake(recorded, bug):
    import replay_fp64

    chk = replay_fp64.Checker()
    replay_fp64.replay([c[:3] for c in recorded], FakeKernels(bug), chk, [c[3] for c in recorded], device="cpu")
    print(chk.table(str(bug)))
    return chk


def test_replay_layout_is_the_engines(recorded):
    """The recording keeps the engine's layout: strided segment_sum outputs and wgrad operands, and chg_linear
    with ``residual is y`` and a ``y_rows`` scatter."""
    seg = [s for n, s, _, _ in recorded if n == "segment_sum" and s[4].stride(0) > s[4].shape[1]]
    wg = [s for n, s, _, _ in recorded if n == "wgrad" and s[2].stride(0) > s[2].shape[1]]
    lin = [s for n, s, _, _ in recorded if n == "linear" and s[3] is not None and s[6] is not None
           and s[3].data_ptr() == s[4].data_ptr()]
    assert seg and wg and lin, (len(seg), len(wg), len(lin))
    assert {s[4].stride(0) for s in seg} == {256} and {s[2].stride(0) for s in wg} == {128}


def test_replay_passes_the_unplanted_fake(recorded):
    chk = _replay_fake(recorded, None)
    assert not chk.failures, "\n".join(chk.failures[:20])
    assert {"segment_sum", "linear", "wgrad", "atom_conv_fwd"} <= chk.kernels


@pytest.mark.parametrize("bug", PLANTED)
def test_replay_flags_a_planted_bug(recorded, bug):
    """Each planted bug is flagged, on the kernel it was planted in and on no other."""
    chk = _replay_fake(recorded, bug)
    kernel = bug.split()[0]
    assert chk.failures, f"{bug}: not flagged"
    assert all(f.startswith(kernel + " ") for f in chk.failures), "\n".join(chk.failures[:20])
