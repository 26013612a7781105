"""-m gpu: every kernel call of engine runs at production sizes, replayed through the CUDA library under the default
dispatch and checked against an fp64 evaluation of its specification (tests/replay_fp64.py).

The mixed batch puts two rattled LiMnO2 supercells (144 and 480 atoms, 84-88 neighbours per atom) between random cells
and a cell without edges, so that the persistent kernels run several tiles per CTA, segments span several 16-row
strips and the virial reduction sees blocks inside one graph and across graphs; ``test_mixed_batch_covers_the_edges``
asserts these properties of the batch itself.  The high-coordination batch of tests/dense_cells.py (rattled diamond
and a 1.1 A simple cubic H/Li cell: segments of 704 edges, 163 bond-graph rows and 6 806 angles per atom, longer than
a tile and than a persistent CTA's share) runs through the same tests: the inference recording is parametrized over
both batches, and the coverage, training and determinism tests check one batch after the other.  The inference
recording and its fp64 references are cached per batch (five implementation slots replay it); the other runs are
checked call by call as they are recorded."""
import dense_cells
import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights

pytestmark = pytest.mark.gpu

N_SM = 132  # H100 SXM
WS_TILE, FFMA_TILE, STRIP, VIRIAL_BLOCK = 128, 64, 16, 256  # csrc/gated_ws.cu, gated.cu, geometry.cu
WS_MIN_ROWS = 4096  # default ws_min_rows: the fused warp-specialised kernels run from this many rows


def _mixed_graphs(**cut):
    rand = graphgen.random_graphs(4, 10, 40, 9900, **cut)
    h2 = graphgen.make_crystal_graph([1, 1], [[0.0, 0.0, 0.0], [0.5, 0.5, 0.5]], 20.0 * np.eye(3), graph_id="h2", **cut)
    big = [graphgen.make_crystal_graph(*graphgen.limno2_structure(sc, 0.02, seed), graph_id=f"limno2{sc}", **cut)
           for sc, seed in (((3, 3, 2), 1), ((5, 4, 3), 2))]
    return [rand[0], big[0], h2, rand[1], rand[2], big[1], rand[3]]


def _packed(w, hp=None):
    return pack_weights({k: torch.as_tensor(v) for k, v in w.items()}, hp, device="cpu")


def _with_refs(calls):
    import replay_fp64

    return [(name, snap, outs) for name, snap, outs in calls], [replay_fp64.reference64(n, s) for n, s, _ in calls]


def _replay(calls, refs=None, options=None, title=""):
    import replay_fp64

    from chgnet_b200._lib import CudaKernels

    K = CudaKernels()
    chk = replay_fp64.Checker()
    try:
        for k, v in (options or {}).items():
            K.set_option(k, v)
        replay_fp64.replay(calls, K, chk, refs)
    finally:
        K.set_option("linear_impl", 3)
        K.set_option("gated_impl", 3)
    chk.assert_ok(title)
    return chk


def _streamed(rec):
    """Replay and check every call of the recorder ``rec`` as it is recorded (see replay_fp64.StreamedCalls)."""
    import replay_fp64

    from chgnet_b200._lib import CudaKernels

    chk = replay_fp64.Checker()
    rec.calls = replay_fp64.StreamedCalls(CudaKernels(), chk)
    return chk


@pytest.fixture(scope="module")
def mixed_graphs():
    return _mixed_graphs()


@pytest.fixture(scope="module")
def dense_graphs():
    return dense_cells.dense_graphs()


def _inference_calls(weights, graphs, calls=None):
    """The kernel calls of an inference run (forces, stress, magmoms, features) on ``graphs``."""
    from kernel_replay import RecordingKernels

    rec = RecordingKernels()
    if calls is not None:
        rec.calls = calls
    Engine(_packed(weights), rec).run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True,
                                      need_atom_fea=True, need_crystal_fea=True)
    return rec.calls


@pytest.fixture(scope="module", params=["mixed", "dense"])
def inference(request, weights030):
    return _with_refs(_inference_calls(weights030, request.getfixturevalue(f"{request.param}_graphs")))


def _longest(ptr):
    ptr = ptr.long()
    return int((ptr[1:] - ptr[:-1]).max())


def test_mixed_batch_covers_the_edges(mixed_graphs, dense_graphs):
    """Both batches: ragged last tiles; the mixed batch several tiles per persistent CTA, segments across strips and
    virial blocks inside and across graphs; the dense batch segments longer than a tile."""
    b = build_batch(dense_graphs, "cpu")
    ed, a = b.n_edges, b.n_angles
    assert ed % WS_TILE and a % WS_TILE, (ed, a)
    assert ed >= WS_MIN_ROWS and a >= WS_MIN_ROWS, (ed, a)  # the default dispatch runs the gated_ws kernels
    assert _longest(b.ptr_c) > 2 * WS_TILE, "an AtomConv segment longer than 256 rows"
    assert _longest(b.ptr_is) > WS_TILE, "a BondConv segment longer than a tile"
    lo, hi = b.ptr_is.long()[:-1], b.ptr_is.long()[1:]
    assert int(((hi - 1) // STRIP - lo // STRIP + 1)[hi > lo].max()) >= 3, "a BondConv segment spanning 3 strips"
    assert _longest(b.ptr_x) > 4096, "angles of one atom: more than 4096 items"
    assert bool((b.ptr_c.long()[1:] == b.ptr_c.long()[:-1]).any()), "an atom without edges"
    print(f"dense batch: {b.n_atoms} atoms, {ed} edges, {a} angles; longest ptr_c {_longest(b.ptr_c)}, "
          f"ptr_is {_longest(b.ptr_is)}, ptr_x {_longest(b.ptr_x)}")

    b = build_batch(mixed_graphs, "cpu")
    ed, a = b.n_edges, b.n_angles
    assert ed % WS_TILE and a % WS_TILE, (ed, a)
    # the warp-specialised fused kernels: at least 2 tiles per persistent CTA; FFMA persistent kernels iterate too
    assert -(-ed // WS_TILE) >= 2 * N_SM and -(-a // WS_TILE) >= 2 * N_SM, (ed, a)
    assert -(-a // FFMA_TILE) > 2 * N_SM
    ptr = b.ptr_c.long()
    lo, hi = ptr[:-1], ptr[1:]
    full = hi > lo
    assert bool((~full).any()), "an atom without edges"
    assert int(((hi - 1) // STRIP - lo // STRIP + 1)[full].max()) >= 3, "a segment spanning 3 strips"
    assert bool((full & (lo % STRIP == 0) & (lo > 0)).any()), "a segment starting on a strip boundary"
    graph_of_edge = b.owner.long()[b.center.long()]
    blocks = [graph_of_edge[s : s + VIRIAL_BLOCK] for s in range(0, ed, VIRIAL_BLOCK)]
    assert any(bool((g == g[0]).all()) for g in blocks) and any(bool((g != g[0]).any()) for g in blocks)
    print(f"mixed batch: {b.n_atoms} atoms, {ed} edges, {b.n_bonds} bonds, {a} angles, {b.n_short} bond-graph bonds")


# the implementation slots of test_kernels_gpu.py::test_every_kernel_matches_its_spec, with its ids; ws_min_rows stays
# at its default, so the tensor-core kernels run where they run in production
@pytest.mark.parametrize("linear_impl,gated_impl", [(3, 3), (3, 0), (1, 0), (0, 1), (2, 2)],
                         ids=["defaults: linear=tcgen05-ws,gated=fused-tcgen05-ws", "linear=tcgen05-ws,gated=ffma4x8",
                              "linear=tcgen05,gated=ffma4x8", "linear=ffma,gated=tcgen05", "linear=tcgen05+tma,gated=ffma8x8"])
def test_inference_at_size_matches_fp64(inference, linear_impl, gated_impl):
    from kernel_replay import INFER_KERNELS

    calls, refs = inference
    chk = _replay(calls, refs, dict(linear_impl=linear_impl, gated_impl=gated_impl), f"inference {linear_impl}/{gated_impl}")
    assert chk.kernels == INFER_KERNELS, sorted(chk.kernels)


def test_training_step_at_size_matches_fp64(weights030, mixed_graphs, dense_graphs):
    """Energy / magmom step, then a step with force and stress seeds: every training and second-order kernel, on the
    mixed and on the dense batch."""
    from kernel_replay import TRAIN_KERNELS, RecordingKernels

    for title, graphs in (("mixed", mixed_graphs), ("dense", dense_graphs)):
        rec = RecordingKernels()
        chk = _streamed(rec)
        eng = Engine(_packed(weights030), rec)
        n, nb = sum(g.atomic_number.shape[0] for g in graphs), len(graphs)
        gen = torch.Generator().manual_seed(12)
        out = eng.run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True, train=True)
        eng.param_grads(out, torch.randn(nb, generator=gen), torch.randn(n, generator=gen))
        out = eng.run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True, train=True)
        eng.input_grads(out, record=True)
        eng.param_grads(out, torch.randn(nb, generator=gen), torch.randn(n, generator=gen),
                        torch.randn(n, 3, generator=gen), torch.randn(nb, 3, 3, generator=gen))
        chk.assert_ok(f"training step, {title} batch")
        assert TRAIN_KERNELS <= chk.kernels, (title, sorted(TRAIN_KERNELS - chk.kernels))


def test_without_layernorm_at_size_matches_fp64(weights030):
    """v0.2.0-shaped weights (no LayerNorm, 9 + 9 basis functions, mlp_out bias, uncompacted bonds) on the mixed batch:
    the use_ln = false epilogues of the fused kernels at size."""
    from kernel_replay import RecordingKernels

    from oracle import chgnet_oracle as orc

    args = dict(num_radial=9, num_angular=9, gMLP_norm=None, readout_norm=None, mlp_out_bias=True, cutoff_coeff=5)
    w = orc.random_weights(3, args)
    w = {k: v for k, v in w.items() if k != "mlp.layers.4.weight" and k != "mlp.layers.4.bias"}
    w["mlp.layers.5.weight"], w["mlp.layers.5.bias"] = w.pop("mlp.layers.7.weight"), w.pop("mlp.layers.7.bias")
    pw = _packed(w, dict(atom_graph_cutoff=5.0, cutoff_coeff=5))
    assert not pw.hp.use_ln
    rec = RecordingKernels()
    chk = _streamed(rec)
    Engine(pw, rec).run(build_batch(_mixed_graphs(atom_graph_cutoff=5.0), "cpu", compact_bonds=False), need_grad=True,
                        need_magmom=True)
    chk.assert_ok("no LayerNorm")
    assert {"atom_conv_fused", "bond_conv_fused", "angle_update_fwd"} <= chk.kernels


def _second_order_recorder():
    import replay_fp64
    from kernel_replay import RecordingKernels

    from oracle.elastic import ElasticSpecKernels

    class Recorder(RecordingKernels, ElasticSpecKernels):
        recorded = replay_fp64.ALL_OUT_ARGS

    return Recorder()


@pytest.mark.parametrize("kind", ["hessian_vector_products", "second_derivatives"])
def test_second_derivatives_at_size_match_fp64(weights030, kind):
    """8 copies of the 144-atom LiMnO2 cell: Hessian-vector products, and strain second derivatives with
    position-only, strain-only and mixed directions."""
    z, frac, lat = graphgen.limno2_structure((3, 3, 2), 0.02, 3)
    g = graphgen.make_crystal_graph(z, frac, lat)
    copies, n = 8, len(z)
    gen = torch.Generator().manual_seed(13)
    v = torch.randn(copies * n, 3, generator=gen)
    rec = _second_order_recorder()
    chk = _streamed(rec)
    eng = Engine(_packed(weights030), rec)
    b = build_batch([g] * copies, "cpu")
    if kind == "hessian_vector_products":
        eng.hessian_vector_products(b, v)
        want = {"bond_basis_hvp", "angle_basis_hvp", "edge_tangent_bwd"}
    else:
        w = torch.randn(copies, 3, 3, generator=gen)
        v[: 3 * n] = 0.0  # copies 0-2: strain only
        w[3:6] = 0.0  # copies 3-5: position only; 6-7: mixed
        eng.second_derivatives(b, v, w)
        want = {"bond_basis_hvp", "angle_basis_hvp", "edge_tangent_bwd_virial"}
    chk.assert_ok(kind)
    assert want <= chk.kernels, sorted(chk.kernels)


def test_fused_and_wgrad_are_deterministic_at_size(weights030, mixed_graphs, dense_graphs):
    """The header's "fixed order: deterministic": the fused message + aggregation kernels under the default dispatch,
    and chg_wgrad under both implementations, give bitwise equal results on a second call, on both batches."""
    import replay_fp64
    from kernel_replay import RecordingKernels

    from chgnet_b200._lib import CudaKernels

    def twice(K, name, snap, outs):
        res = []
        for _ in range(2):
            args = replay_fp64.place(snap)[0]
            getattr(K, name)(*args)
            torch.cuda.synchronize()
            res.append([args[i] for i in outs])
        for i, x, y in zip(outs, *res):
            assert torch.equal(x, y), f"{name} out[{i}] differs between two identical calls"

    class Fused(list):  # keeps only the fused message + aggregation calls
        def append(self, call):
            if call[0] in ("atom_conv_fused", "bond_conv_fused"):
                super().append(call)

    def rows(snap):  # m of chg_wgrad: x_rows, else g_rows, else the rows of x
        return next(t.shape[0] for t in (snap[4], snap[5], snap[0]) if t is not None)

    class LargeWgrad(list):  # keeps only the chg_wgrad calls in the tensor-core kernel's range (>= 4096 rows)
        def append(self, call):
            if call[0] == "wgrad" and rows(call[1]) >= 4096:
                super().append(call)

    K = CudaKernels()
    for graphs in (mixed_graphs, dense_graphs):
        fused = _inference_calls(weights030, graphs, Fused())
        assert {c[0] for c in fused} == {"atom_conv_fused", "bond_conv_fused"}
        for name, snap, outs in fused:
            twice(K, name, snap, outs)
        del fused
        rec = RecordingKernels()
        rec.calls = LargeWgrad()
        eng = Engine(_packed(weights030), rec)
        n, nb = sum(g.atomic_number.shape[0] for g in graphs), len(graphs)
        gen = torch.Generator().manual_seed(14)
        out = eng.run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True, train=True)
        eng.param_grads(out, torch.randn(nb, generator=gen), torch.randn(n, generator=gen))
        wgrad = list(rec.calls)
        assert wgrad
        try:
            for impl in (1, 0):
                K.set_option("wgrad_impl", impl)
                for name, snap, outs in wgrad:
                    twice(K, name, snap, outs)
        finally:
            K.set_option("wgrad_impl", 1)
