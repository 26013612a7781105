"""Training step on the kernel engine (reference chgnet/trainer/trainer.py).

Mirrors the pieces of the reference ``Trainer`` that sit on the hot path of a fine-tuning step
(trainer.py:398-411): prediction -> ``CombinedLoss`` (779-869) -> ``loss.backward()`` ->
``optimizer.step()``, with the same constructor vocabulary (``targets``, ``criterion``,
``energy_loss_ratio`` ..., ``optimizer="Adam"``, ``learning_rate``, ``delta``,
``allow_missing_labels``).

What is covered (DESIGN.md §9): every ``targets`` string of the reference ("e", "ef", "em", "efs",
"efsm"), MSE / MAE / Huber with NaN-masked missing labels, Adam as one fused kernel over a flat
parameter buffer, data-parallel training with ONE all-reduce of the flat gradient buffer per step
(SURVEY.md §8e).  Losses on forces / stresses go through the second-order pass of the engine
(``Engine._second_order``: tangent pass + reverse over (primal, tangent)), which replaces autograd's
double backward (model.py:518-535 ``create_graph=True``).

The loss normalisation follows the reference exactly for one process (``nn.MSELoss`` means over
the batch); across ranks the means are over the GLOBAL batch: the per-term numerators and counts
are all-reduced before the seeds are formed, and the gradient buffers are summed.
"""
from __future__ import annotations

from collections.abc import Sequence
from dataclasses import dataclass

import torch
from torch import Tensor

from chgnet_b200.weights import GradFlattenMap, RepackMap, unpack_grads

_KIND = {"MSE": 0, "mse": 0, "MAE": 1, "mae": 1, "l1": 1, "Huber": 2}


@dataclass
class LossConfig:
    target_str: str = "e"
    criterion: str = "MSE"
    energy_loss_ratio: float = 1.0
    force_loss_ratio: float = 1.0
    stress_loss_ratio: float = 0.1
    mag_loss_ratio: float = 0.1
    delta: float = 0.1

    def __post_init__(self) -> None:
        if self.criterion not in _KIND:
            raise NotImplementedError(self.criterion)  # same as trainer.py:763
        if not set(self.target_str) <= set("efsm") or "e" not in self.target_str:
            raise ValueError(f"Invalid targets={self.target_str!r}")


def _all_reduce(t: Tensor, group) -> None:
    """SUM over the ranks of ``group`` (None = default group; False = this rank only)."""
    import torch.distributed as dist

    if group is False:
        return
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, group=group)


def loss_and_seeds(K, cfg: LossConfig, preds: dict[str, Tensor], targets: dict[str, Tensor], group=None) -> tuple[dict, dict]:
    """CombinedLoss (trainer.py:779-869) on the device.

    ``preds`` / ``targets``: flat-able tensors per key of ``cfg.target_str`` (e [B], f [N,3], s [B,3,3],
    m [N]); NaN targets are missing labels.  Returns (report, seeds): ``report`` holds python floats
    (loss, X_MAE, X_MAE_size per term), ``seeds[key]`` = d loss / d preds[key].  With an initialised
    process group the means are over the global batch.
    """
    kind = _KIND[cfg.criterion]
    keys = [k for k in "efsm" if k in cfg.target_str and preds.get(k) is not None and targets.get(k) is not None]
    ratio = {"e": cfg.energy_loss_ratio, "f": cfg.force_loss_ratio, "s": cfg.stress_loss_ratio, "m": cfg.mag_loss_ratio}
    dev = preds["e"].device
    sums = torch.zeros(len(keys), 3, dtype=torch.float64, device=dev)
    raw = {}
    for i, k in enumerate(keys):
        p = preds[k].contiguous()
        raw[k] = torch.empty_like(p)
        K.loss_terms(p.view(-1), targets[k].to(p.dtype).contiguous().view(-1), kind, cfg.delta, raw[k].view(-1), sums[i])
    _all_reduce(sums, group)
    cnt = sums[:, 2].clamp_min(1.0)
    seeds = {k: raw[k] * (ratio[k] / cnt[i]).to(raw[k].dtype) for i, k in enumerate(keys)}
    host = sums.cpu()
    report = {"loss": 0.0}
    for i, k in enumerate(keys):
        n = max(float(host[i, 2]), 1.0)
        report["loss"] += ratio[k] * float(host[i, 0]) / n
        report[f"{k}_MAE"], report[f"{k}_MAE_size"] = float(host[i, 1]) / n, int(host[i, 2])
    return report, seeds


def loss_and_grads(engine, batch, cfg: LossConfig, targets: dict[str, Tensor], is_intensive: bool = True,
                   group=None) -> tuple[dict, dict]:
    """One forward (+ force pass) + loss + training reverse pass on an already built batch.

    ``targets``: e [B] (per atom if ``is_intensive``), f [N,3], s [B,3,3] (GPa), m [N], as far as
    ``cfg.target_str`` asks.  Returns (report, packed-layout gradients of THIS rank's graphs under the
    global-batch loss); sum the gradients over ranks to get the global gradient.
    """
    from chgnet_b200.engine import EV_A3_TO_GPA

    K = engine.K
    second = "f" in cfg.target_str or "s" in cfg.target_str
    out = engine.run(batch, need_grad=True, need_magmom="m" in cfg.target_str, train=True)
    if second:
        engine.input_grads(out, record=True)
    n = torch.tensor(batch.atoms_per_graph, device=out.energy.device, dtype=out.energy.dtype)
    total = out.energy + out.e_ref
    dt = out.site_e.dtype
    preds = {"e": (total / n if is_intensive else total).to(dt), "m": out.magmom}
    if "f" in cfg.target_str:
        preds["f"] = out.force.to(dt)
    if "s" in cfg.target_str:
        scale = EV_A3_TO_GPA / batch.volume.to(torch.float64)
        preds["s"] = (out.virial.view(-1, 3, 3) * scale[:, None, None]).to(dt)
    report, seeds = loss_and_seeds(K, cfg, preds, targets, group)
    seed_e = seeds["e"] / n.to(dt) if is_intensive else seeds["e"]
    return report, engine.param_grads(out, seed_e.contiguous(), seeds.get("m"), seeds.get("f"), seeds.get("s"))


class Trainer:
    """Fine-tuning loop on the CUDA kernel path (reference Trainer, trainer.py:37-411).

    >>> trainer = Trainer(model, targets="em", optimizer="Adam", criterion="MSE", learning_rate=1e-3)
    >>> report = trainer.train_step(graphs, {"e": e_labels, "m": [m_0, m_1, ...]})
    """

    def __init__(self, model, *, targets: str = "e", energy_loss_ratio: float = 1, force_loss_ratio: float = 1,
                 stress_loss_ratio: float = 0.1, mag_loss_ratio: float = 0.1, optimizer: str = "Adam",
                 criterion: str = "MSE", learning_rate: float = 1e-3, weight_decay: float = 0.0,
                 betas: tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, delta: float = 0.1,
                 scheduler: str = "CosLR", scheduler_params: dict | None = None, epochs: int = 50,
                 process_group=None, **_: object) -> None:
        if optimizer != "Adam":
            raise NotImplementedError("chgnet_b200.Trainer implements optimizer='Adam' (the reference default)")
        self.trainer_args = dict(targets=targets, energy_loss_ratio=energy_loss_ratio, force_loss_ratio=force_loss_ratio,
                                 stress_loss_ratio=stress_loss_ratio, mag_loss_ratio=mag_loss_ratio, optimizer=optimizer,
                                 criterion=criterion, learning_rate=learning_rate, weight_decay=weight_decay, betas=betas,
                                 eps=eps, delta=delta, scheduler=scheduler, scheduler_params=scheduler_params, epochs=epochs)
        self.training_history: list[dict] = []
        self.schedule = LRSchedule(scheduler, learning_rate, epochs, scheduler_params)
        self.epochs = epochs
        self.model = model
        self.cfg = LossConfig(targets, criterion, energy_loss_ratio, force_loss_ratio, stress_loss_ratio,
                              mag_loss_ratio, delta)
        if "m" in targets and model.n_conv < 2:
            raise ValueError(f"n_conv={model.n_conv}: magnetic moments are read after block n_conv - 1, which a model "
                             f"with one block does not have (targets={targets!r})")
        self.lr, self.weight_decay, self.betas, self.eps = learning_rate, weight_decay, betas, eps
        self.group = process_group
        self.step_count = 0
        # one flat fp32 buffer holds every trainable parameter; the nn.Parameters become views of it,
        # so state_dict() stays the single source of truth and Adam is ONE kernel launch
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
        self.names = [n for n, _ in named]
        self.shapes = [tuple(p.shape) for _, p in named]
        self.sizes = [p.numel() for _, p in named]
        # every parameter starts on a 64-byte boundary (the kernels read weights as float4); the
        # padding stays zero under Adam (zero gradient, zero moments)
        self.offsets, off = [], 0
        for sz in self.sizes:
            self.offsets.append(off)
            off += (sz + 15) // 16 * 16
        dev = named[0][1].device
        self.flat = torch.zeros(off, dtype=torch.float32, device=dev)
        for (_, p), o, sz in zip(named, self.offsets, self.sizes):
            self.flat[o:o + sz] = p.detach().reshape(-1)
            p.data = self.flat[o:o + sz].view(p.shape)
        self.flat_grad = torch.zeros_like(self.flat)
        self.exp_avg = torch.zeros_like(self.flat)
        self.exp_avg_sq = torch.zeros_like(self.flat)
        model.mark_params_updated()
        self._repack: RepackMap | None = None  # in-place refresh of the packed kernel weights (built on first use)
        self._gflat: GradFlattenMap | None = None  # packed-layout gradients -> flat buffer in one gather

    # ------------------------------------------------------------------
    def _targets(self, targets: dict, n_list: Sequence[int], device) -> dict[str, Tensor]:
        """reference label layout (dataset.py:763-788: e [B], f / m lists per graph, s list of [3,3]) ->
        flat device tensors; None / NaN = missing labels (trainer.py:846-851)"""
        def per_graph(vals, shape_of):
            parts = [torch.full(shape_of(n), float("nan")) if v is None else torch.as_tensor(v, dtype=torch.float32).reshape(shape_of(n))
                     for n, v in zip(n_list, vals)]
            return torch.cat(parts).to(device)

        out = {"e": torch.as_tensor(targets["e"], dtype=torch.float32).reshape(-1).to(device)}
        if "f" in self.cfg.target_str:
            out["f"] = per_graph(targets["f"], lambda n: (n, 3))
        if "s" in self.cfg.target_str:
            out["s"] = per_graph(targets["s"], lambda n: (1, 3, 3))
        if "m" in self.cfg.target_str:
            out["m"] = per_graph(targets["m"], lambda n: (n,))
        return out

    def flatten_grads(self, grads: dict[str, Tensor]) -> Tensor:
        for name, o, sz in zip(self.names, self.offsets, self.sizes):
            self.flat_grad[o:o + sz] = grads[name].reshape(-1)
        return self.flat_grad

    def flatten_packed_grads(self, G: dict) -> Tensor:
        """``Engine.param_grads`` output -> ``self.flat_grad`` with one concatenation + one gather (the index map is
        derived once from ``unpack_grads`` itself, so both routes agree element for element)."""
        if self._gflat is None or not self._gflat.matches(G):
            self._gflat = GradFlattenMap(G, self.model.state_dict(), self.names, self.offsets, self.sizes, self.flat.numel())
        return self._gflat.flatten(G, self.flat_grad)

    def refresh_packed_weights(self) -> None:
        """After the fused Adam step changed the flat buffer: refresh the engine's packed weights in place (one gather)
        instead of re-packing ~130 tensors in Python.  The inference-side packed blob (chg_forward) is dropped and rebuilt
        on the next prediction."""
        model = self.model
        model._native_key = None
        eng = model._engine
        if eng is None:
            model.mark_params_updated()
            return
        if self._repack is None or self._repack.pw is not eng.pw:
            self._repack = RepackMap(eng.pw, model.state_dict(), model.model_args, self.names, self.offsets, self.flat)
        self._repack.refresh(self.flat)
        model._mark_engine_current()

    def grads_by_name(self) -> dict[str, Tensor]:
        """views of the (all-reduced) flat gradient buffer, one per parameter"""
        return {n: self.flat_grad[o:o + sz].view(sh) for n, o, sz, sh in zip(self.names, self.offsets, self.sizes, self.shapes)}

    def train_step(self, graphs, targets: dict) -> dict:
        """prediction -> CombinedLoss -> parameter gradients -> (all-reduce) -> Adam; returns the report."""
        from chgnet_b200.batch import build_batch

        model = self.model
        engine = model._get_engine()
        compact = not any(gp.extra["bo"] is not None for gp in engine.pw.bond)
        batch = build_batch(graphs, model.device, with_reverse=True, compact_bonds=compact)
        tg = self._targets(targets, batch.atoms_per_graph, model.device)
        report, G = loss_and_grads(engine, batch, self.cfg, tg, model.is_intensive, self.group)
        flat_grad = self.flatten_packed_grads(G)
        _all_reduce(flat_grad, self.group)  # the one collective of the step (SURVEY.md §8e)
        self.step_count += 1
        engine.K.adam_step(self.flat, flat_grad, self.exp_avg, self.exp_avg_sq, self.lr, self.betas[0],
                           self.betas[1], self.eps, self.weight_decay, self.step_count)
        self.refresh_packed_weights()
        return report

    # ------------------------------------------------------------------ checkpoint / resume (trainer.py:614-688)
    def save(self, filename: str = "training_result.pth.tar") -> None:
        """model (reference ``as_dict`` layout: loadable by ``CHGNet.from_file`` here and in the reference),
        optimizer moments, schedule position, history, constructor arguments"""
        by_name = lambda buf: {n: buf[o:o + sz].view(sh).detach().cpu().clone()  # noqa: E731
                               for n, o, sz, sh in zip(self.names, self.offsets, self.sizes, self.shapes)}
        state = {"model": {"model_args": self.model.model_args,
                           "state_dict": {k: v.detach().cpu().clone() for k, v in self.model.state_dict().items()}},
                 "optimizer": {"step": self.step_count, "exp_avg": by_name(self.exp_avg), "exp_avg_sq": by_name(self.exp_avg_sq)},
                 "scheduler": {"t": self.schedule.t, "lr": self.lr},
                 "training_history": self.training_history, "trainer_args": self.trainer_args}
        torch.save(state, filename)

    @classmethod
    def load(cls, path: str, device=None, **overrides):
        """Rebuild a trainer (model on ``device``, default: CUDA) and resume where ``save`` stopped."""
        from chgnet_b200.model import CHGNet

        state = torch.load(path, map_location="cpu", weights_only=False)
        model = CHGNet.from_dict(state["model"])
        model = model.to(device if device is not None else "cuda")
        trainer = cls(model, **{**state["trainer_args"], **overrides})
        opt = state["optimizer"]
        trainer.step_count = int(opt["step"])
        for n, o, sz in zip(trainer.names, trainer.offsets, trainer.sizes):
            trainer.exp_avg[o:o + sz] = opt["exp_avg"][n].reshape(-1).to(trainer.exp_avg.device)
            trainer.exp_avg_sq[o:o + sz] = opt["exp_avg_sq"][n].reshape(-1).to(trainer.exp_avg.device)
        trainer.schedule.t, trainer.lr = int(state["scheduler"]["t"]), float(state["scheduler"]["lr"])
        trainer.training_history = list(state["training_history"])
        return trainer

    def scheduler_step(self) -> float:
        """advance the learning-rate schedule by one tick (the reference ticks 10 times per epoch,
        trainer.py:413-415); returns the new learning rate"""
        self.lr = self.schedule.step()
        return self.lr

    def train(self, loader, epochs: int | None = None) -> list[dict]:
        """``loader`` (a sized iterable) yields (graphs, targets) like the reference's collate_graphs
        batches (dataset.py:763-788); the schedule is advanced every 1/10 of an epoch."""
        history = []
        n = len(loader)
        ticks = {int(k * n // 10) for k in range(1, 11)}  # np.arange(1, 11) * len(loader) // 10
        for _ in range(self.epochs if epochs is None else epochs):
            for idx, (graphs, targets) in enumerate(loader):
                history.append(self.train_step(graphs, targets))
                self.training_history.append(history[-1])
                if idx + 1 in ticks:
                    self.scheduler_step()
        return history


class LRSchedule:
    """Closed forms of the reference's schedulers (trainer.py:165-205): CosineAnnealingLR with
    ``T_max = 10 * epochs`` and ``eta_min = decay_fraction * lr`` (default), ExponentialLR, MultiStepLR."""

    def __init__(self, kind: str, lr: float, epochs: int, params: dict | None = None) -> None:
        import math

        self.lr0, self.t, self._math = lr, 0, math
        params = dict(params or {})
        if kind in {"CosineAnnealingLR", "CosLR", "Cos", "cos"}:
            self.kind, self.t_max = "cos", 10 * epochs
            self.eta_min = params.get("decay_fraction", 1e-2) * lr
        elif kind in {"ExponentialLR", "Exp", "Exponential"}:
            self.kind, self.gamma = "exp", params.get("gamma", 0.98)
        elif kind in {"MultiStepLR", "multistep"}:
            self.kind = "multistep"
            self.milestones = sorted(params.get("milestones", [4 * epochs, 6 * epochs, 8 * epochs, 9 * epochs]))
            self.gamma = params.get("gamma", 0.3)
        else:
            raise NotImplementedError(kind)

    def value(self, t: int) -> float:
        if self.kind == "cos":
            return self.eta_min + (self.lr0 - self.eta_min) * (1 + self._math.cos(self._math.pi * t / self.t_max)) / 2
        if self.kind == "exp":
            return self.lr0 * self.gamma**t
        return self.lr0 * self.gamma ** sum(1 for m in self.milestones if m <= t)

    def step(self) -> float:
        self.t += 1
        return self.value(self.t)
