"""-m gpu: every C-ABI kernel, called through ctypes with the exact arguments of a real
forward + reverse pass, against its torch specification (oracle/kernel_specs.py)."""
import numpy as np
import pytest
import torch

from chgnet_b200 import graphgen
from chgnet_b200.batch import build_batch
from chgnet_b200.engine import Engine
from chgnet_b200.weights import pack_weights

pytestmark = pytest.mark.gpu


def _record(weights, graphs, **kw):
    from kernel_replay import RecordingKernels

    sd = {k: torch.as_tensor(v) for k, v in weights.items()}
    pw = pack_weights(sd, None, device="cpu")
    rec = RecordingKernels()
    Engine(pw, rec).run(build_batch(graphs, "cpu"), **kw)
    return rec.calls


@pytest.fixture(scope="module")
def recorded(weights030):
    """The calls of a forward + reverse pass and their fp64 references (tests/replay_fp64.py)."""
    import replay_fp64

    graphs = graphgen.random_graphs(3, 10, 16, 9300)
    calls = _record(weights030, graphs, need_grad=True, need_magmom=True, need_atom_fea=True, need_crystal_fea=True)
    return calls, [replay_fp64.reference64(name, snap) for name, snap, _ in calls]


# ids are the stable names of the implementation slots (option values); on sm_90a every tensor-core slot is a wgmma kernel
@pytest.mark.parametrize("linear_impl,gated_impl", [(3, 3), (3, 0), (1, 0), (0, 1), (2, 2)],
                         ids=["defaults: linear=tcgen05-ws,gated=fused-tcgen05-ws", "linear=tcgen05-ws,gated=ffma4x8",
                              "linear=tcgen05,gated=ffma4x8", "linear=ffma,gated=tcgen05", "linear=tcgen05+tma,gated=ffma8x8"])
def test_every_kernel_matches_its_spec(recorded, linear_impl, gated_impl):
    """Both implementations of every entry point (wgmma 3xTF32 and FFMA) against the fp64 spec."""
    import replay_fp64

    from chgnet_b200._lib import CudaKernels

    K = CudaKernels()
    K.set_option("linear_impl", linear_impl)
    K.set_option("gated_impl", gated_impl)
    K.set_option("ws_min_rows", 0)  # the recorded graphs are small: run the tensor-core kernels on them anyway
    try:
        chk = replay_fp64.Checker()
        calls, refs = recorded
        replay_fp64.replay(calls, K, chk, refs)
        chk.assert_ok(f"linear_impl={linear_impl}, gated_impl={gated_impl}")
        assert chk.kernels == __import__("kernel_replay").INFER_KERNELS, sorted(chk.kernels)
    finally:
        K.set_option("linear_impl", 3)
        K.set_option("gated_impl", 3)
        K.set_option("ws_min_rows", 4096)


def test_every_training_kernel_matches_its_spec(weights030):
    """Training reverse pass (parameter gradients): every call of a real train step, replayed."""
    import kernel_replay
    import replay_fp64
    from chgnet_b200._lib import CudaKernels
    from kernel_replay import RecordingKernels

    graphs = graphgen.random_graphs(3, 10, 16, 9500)
    sd = {k: torch.as_tensor(v) for k, v in weights030.items()}
    pw = pack_weights(sd, None, device="cpu")
    rec = RecordingKernels()
    eng = Engine(pw, rec)
    out = eng.run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True, train=True)
    gen = torch.Generator().manual_seed(11)
    n_atoms = sum(g.atomic_number.shape[0] for g in graphs)
    eng.param_grads(out, torch.randn(len(graphs), generator=gen), torch.randn(n_atoms, generator=gen))
    # and a step with force / stress seeds: the second-order kernels
    out = eng.run(build_batch(graphs, "cpu"), need_grad=True, need_magmom=True, train=True)
    eng.input_grads(out, record=True)
    eng.param_grads(out, torch.randn(len(graphs), generator=gen), torch.randn(n_atoms, generator=gen),
                    torch.randn(n_atoms, 3, generator=gen), torch.randn(len(graphs), 3, 3, generator=gen))
    chk = replay_fp64.Checker()
    replay_fp64.replay(rec.calls, CudaKernels(), chk)
    chk.assert_ok("training")
    assert kernel_replay.TRAIN_KERNELS <= chk.kernels, sorted(chk.kernels)


def test_loss_terms_and_adam_match_torch():
    """chg_loss_terms vs torch.nn.{MSE,L1,Huber}Loss with NaN masks (trainer.py:797-867) and
    chg_adam_step vs torch.optim.Adam (trainer.py:178-189)."""
    from chgnet_b200._lib import CudaKernels

    K = CudaKernels()
    g = torch.Generator(device="cuda").manual_seed(2)
    pred = torch.randn(5000, device="cuda", generator=g)
    target = pred + 0.3 * torch.randn(5000, device="cuda", generator=g)
    target[::7] = float("nan")
    valid = ~torch.isnan(target)
    for kind, crit in ((0, torch.nn.MSELoss()), (1, torch.nn.L1Loss()), (2, torch.nn.HuberLoss(delta=0.1))):
        p = pred.clone().requires_grad_(True)
        loss = crit(target[valid], p[valid])
        loss.backward()
        g_pred, sums = torch.empty_like(pred), torch.zeros(3, dtype=torch.float64, device="cuda")
        K.loss_terms(pred, target, kind, 0.1, g_pred, sums)
        n = float(sums[2])
        assert n == float(valid.sum())
        assert float(sums[0]) / n == pytest.approx(float(loss), rel=1e-5)
        assert float(sums[1]) / n == pytest.approx(float((pred - target)[valid].abs().mean()), rel=1e-5)
        assert float((g_pred / n - p.grad).abs().max()) < 1e-7
    p0 = torch.randn(100_003, device="cuda", generator=g)
    ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-3)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for step in range(1, 4):
        grad = torch.randn(p0.shape, device="cuda", generator=g)
        ref.grad = grad.clone()
        opt.step()
        K.adam_step(p, grad, m, v, 1e-2, 0.9, 0.999, 1e-8, 1e-3, step)
        assert float((p - ref.detach()).abs().max()) < 2e-6


# ids are the stable names of the implementation slots (option values); on sm_90a every tensor-core slot is a wgmma kernel
@pytest.mark.parametrize("impl", [3, 2, 1, 0], ids=["tcgen05-ws", "tcgen05+tma", "tcgen05", "ffma"])
def test_linear_large_ragged_calls(impl):
    """chg_linear at the sizes where the tensor-core kernels are dispatched (m >= 4096): ragged
    last tile, every (k, n) the model uses, bias / residual / in-place residual, against fp64."""
    from chgnet_b200._lib import CudaKernels

    K = CudaKernels()
    K.set_option("linear_impl", impl)
    g = torch.Generator(device="cuda").manual_seed(5)
    try:
        for m in (4096, 5001, 70001):
            for k, n in ((64, 128), (64, 256), (128, 64), (64, 64), (64, 192), (128, 128), (256, 64)):
                for has_bias, res_mode in ((True, "none"), (False, "separate"), (True, "inplace")):
                    x = torch.randn(m, k, device="cuda", generator=g)
                    wt = torch.randn(k, n, device="cuda", generator=g) / k ** 0.5
                    bias = torch.randn(n, device="cuda", generator=g) if has_bias else None
                    res = torch.randn(m, n, device="cuda", generator=g) if res_mode != "none" else None
                    want = x.double() @ wt.double()
                    if bias is not None:
                        want += bias.double()
                    if res is not None:
                        want += res.double()
                    y = res if res_mode == "inplace" else torch.full((m, n), float("nan"), device="cuda")
                    K.linear(x, wt, bias, res, y, None, None)
                    torch.cuda.synchronize()
                    err = float((y.double() - want).abs().max())
                    assert err < 5e-5, (impl, m, k, n, has_bias, res_mode, err)
    finally:
        K.set_option("linear_impl", 3)


def test_kernels_without_layernorm_and_small_basis(weights030):
    """v0.2.0-shaped path: no LayerNorm, 9 radial / 9 angular functions, mlp_out bias."""
    import replay_fp64

    from chgnet_b200._lib import CudaKernels
    from oracle import chgnet_oracle as orc

    args = dict(num_radial=9, num_angular=9, gMLP_norm=None, readout_norm=None, mlp_out_bias=True, cutoff_coeff=5)
    w = orc.random_weights(3, args)
    w = {k: v for k, v in w.items() if k != "mlp.layers.4.weight" and k != "mlp.layers.4.bias"}
    w["mlp.layers.5.weight"], w["mlp.layers.5.bias"] = w.pop("mlp.layers.7.weight"), w.pop("mlp.layers.7.bias")
    graphs = graphgen.random_graphs(2, 8, 12, 9400, atom_graph_cutoff=5.0)
    sd = {k: torch.as_tensor(v) for k, v in w.items()}
    from kernel_replay import RecordingKernels

    pw = pack_weights(sd, dict(atom_graph_cutoff=5.0, cutoff_coeff=5), device="cpu")
    assert not pw.hp.use_ln and pw.hp.n_readout_hidden == 2 and pw.hp.num_radial == 9
    rec = RecordingKernels()
    Engine(pw, rec).run(build_batch(graphs, "cpu", compact_bonds=False), need_grad=True, need_magmom=True)
    chk = replay_fp64.Checker()
    replay_fp64.replay(rec.calls, CudaKernels(), chk)
    chk.assert_ok("no LayerNorm, small basis")


def test_segment_sum_strided_output_and_determinism():
    from chgnet_b200._lib import CudaKernels

    K = CudaKernels()
    g = torch.Generator().manual_seed(0)
    n_rows, n_items = 1000, 50000
    owners = torch.sort(torch.randint(0, n_rows, (n_items,), generator=g)).values
    ptr = torch.searchsorted(owners, torch.arange(n_rows + 1)).int().cuda()
    perm = torch.randperm(n_items, generator=g).int().cuda()
    for width in (64, 128):
        data = torch.randn(n_items, width, generator=g).cuda()
        out = torch.zeros(n_rows, 256, device="cuda")
        K.segment_sum(data, perm, ptr, 0, out[:, 64 : 64 + width])
        want = torch.zeros(n_rows, width, dtype=torch.float64).index_add_(0, owners, data[perm.long()].double().cpu())
        assert torch.allclose(out[:, 64 : 64 + width].double().cpu(), want, atol=1e-4)
        assert float(out[:, :64].abs().max()) == 0.0 and float(out[:, 64 + width :].abs().max()) == 0.0
        again = torch.zeros(n_rows, 256, device="cuda")
        K.segment_sum(data, perm, ptr, 0, again[:, 64 : 64 + width])
        assert torch.equal(out, again)  # bitwise reproducible
        K.segment_sum(data, perm, ptr, 1, again[:, 64 : 64 + width])
        assert torch.allclose(again[:, 64 : 64 + width], 2 * out[:, 64 : 64 + width], rtol=1e-6)


def test_bad_arguments_are_reported():
    from chgnet_b200._lib import ChgnetB200Error, CudaKernels

    K = CudaKernels()
    x = torch.zeros(4, 96, device="cuda")
    with pytest.raises(ChgnetB200Error, match="k must be"):
        K.linear(x, torch.zeros(96, 64, device="cuda"), None, None, torch.zeros(4, 64, device="cuda"))
    with pytest.raises(ChgnetB200Error):
        K.linear(torch.zeros(4, 64), torch.zeros(64, 64), None, None, torch.zeros(4, 64))  # CPU tensors


# ids are the stable names of the implementation slots (option values); on sm_90a every tensor-core slot is a wgmma kernel
@pytest.mark.parametrize("wgrad_impl", [1, 0], ids=["tcgen05", "ffma"])
def test_wgrad_large_reduction_matches_fp64(wgrad_impl):
    """chg_wgrad at the sizes where the tensor-core kernel (csrc/wgrad_tc.cu, 3xTF32) takes over (>= 4096 rows): plain,
    SiLU'd and tangent activations, row gathers on either operand, strided operands, column sums - against fp64."""
    from chgnet_b200._lib import CudaKernels

    K = CudaKernels()
    K.set_option("wgrad_impl", wgrad_impl)
    try:
        gen = torch.Generator(device="cuda").manual_seed(5)
        m = 20011  # not a multiple of the 64-row stage
        xs = torch.randn(m, 128, device="cuda", generator=gen)
        x2 = torch.randn(m, 128, device="cuda", generator=gen)
        gs = torch.randn(m, 256, device="cuda", generator=gen)
        perm = torch.randperm(m, device="cuda", generator=gen).int()
        sub = perm[:9000].contiguous()
        silu, dsilu = torch.nn.functional.silu, (lambda t: torch.sigmoid(t) * (1 + t * (1 - torch.sigmoid(t))))
        cases = [
            dict(x=xs[:, :64], g=gs[:, :128], n=128),
            dict(x=xs[:, 64:], g=gs[:, 64:128], n=64, x_silu=True, colsum=True),
            dict(x=xs[:, :64], g=gs[:, 128:], n=128, x2=x2[:, :64]),
            dict(x=xs[:, :64], g=gs[:, :128], n=128, x_rows=sub, colsum=True),
            dict(x=xs[:, 64:], g=gs[:, :64], n=64, g_rows=sub),
        ]
        for c in cases:
            n = c["n"]
            out = torch.empty(64, n, device="cuda")
            cs = torch.empty(n, device="cuda") if c.get("colsum") else None
            K.wgrad(c["x"], c["g"], out, cs, c.get("x_rows"), c.get("g_rows"), c.get("x_silu", False), c.get("x2"))
            torch.cuda.synchronize()
            xr = c["x"].double() if c.get("x_rows") is None else c["x"].double()[c["x_rows"].long()]
            gr = c["g"].double() if c.get("g_rows") is None else c["g"].double()[c["g_rows"].long()]
            if c.get("g_rows") is not None and c.get("x_rows") is None:
                xr = xr[: gr.shape[0]]
            if c.get("x_rows") is not None and c.get("g_rows") is None:
                gr = gr[: xr.shape[0]]
            act = xr
            if c.get("x_silu"):
                act = silu(xr)
            if c.get("x2") is not None:
                act = dsilu(xr) * c["x2"].double()
            want = act.T @ gr
            scale = float(want.abs().max())
            err = float((out.double() - want).abs().max())
            assert err < 3e-5 * scale + 1e-5, (wgrad_impl, c.keys(), err, scale)
            if cs is not None:
                wc = gr.sum(dim=0)
                assert float((cs.double() - wc).abs().max()) < 3e-5 * float(wc.abs().max()) + 1e-4
    finally:
        K.set_option("wgrad_impl", 1)
